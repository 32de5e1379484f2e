"""Ledger of kernel launch variants: one entry per ``__global__`` kernel template in ``model_optimizer_b200/csrc``.

Each C-ABI entry point picks one of several template instantiations at launch time, from the pointer alignment of
its tensors, their shapes and the tuning knobs (``b200q_set_tuning``).  For every kernel this module records:

- ``file``: the source file that defines it;
- ``entry``: the C-ABI entry point(s) that launch it;
- ``variants``: ``(name, condition, test)`` per reachable instantiation, where ``name`` is the demangled name a
  profiler shows without ``void`` and the argument list (``{T}`` stands for any of the three element tags,
  ``b200q::BF16Tag`` / ``F16Tag`` / ``F32Tag``, and ``*`` for any one template argument), ``condition`` what selects
  it, and ``test`` the test module that holds it to the oracle.

``tests/test_dispatch_ledger_cpu.py`` keeps the ledger in step with the sources; ``tests/test_gpu_dispatch_paths.py``
runs every variant whose test is ``DISPATCH`` under ``torch.profiler`` and checks at teardown that each one ran.
"""

import re

DISPATCH = "tests/test_gpu_dispatch_paths.py"
KERNELS_T = "tests/test_gpu_kernels.py"
FUSED_T = "tests/test_gpu_fused_collect_fq.py"
STORE_T = "tests/test_gpu_store_order.py"
ROTATE_T = "tests/test_gpu_rotate.py"
GPTQ_T = "tests/test_gpu_gptq.py"
CALIB_T = "tests/test_gpu_calibrators.py"
SEARCH_T = "tests/test_gpu_search_and_host.py"
E2M1_T = "tests/test_gpu_e2m1_round.py"
HESSIAN_T = "tests/test_gpu_hessian_sweep.py"

_A32 = "x (and y) 32-byte aligned, vec_bytes unset"
_A16 = "a pointer 16- but not 32-byte aligned, or vec_bytes=16"
_L = (1, 2, 4, 8, 16, 32)                         # lanes per quant block: block_size / 16 for 16 .. 512
_B = ("false", "true")


def _fq_variants():
    """fake_quant_kernel<T, VB, UNROLL, KIND, MODE>: KIND 0 INT, 1 FP8 (CUDA or eager rule), 2 FP8 cast (no amax);
    MODE 0 per tensor, 1 per row (vector), 2 per element, 3 per row (CTA tile).  The tile mode runs at unroll 2 when
    the row is a whole number of 512-vector tiles and ew_unroll is 2 (the default), else at unroll 1."""
    out = []
    modes = {0: "one amax (or no amax)", 1: "n_amax > 1, the row (outer) a whole number of vectors, not of tiles",
             2: "n_amax > 1, outer not a multiple of the vector width", 3: "n_amax > 1, the row a whole number of tiles"}
    for vb in (32, 16):
        for kind in (0, 1, 2):
            for mode in ((0,) if kind == 2 else (0, 1, 2, 3)):
                for u in ((2, 1) if mode == 3 else (1, 2, 4)):
                    knob = {1: "ew_unroll=1", 2: "ew_unroll unset", 4: "ew_unroll=4"}[u]
                    if mode == 3:
                        knob = "ew_unroll unset, 512-vector rows" if u == 2 else "256-vector rows, or ew_unroll != 2"
                    out.append((f"b200q::fake_quant_kernel<{{T}}, {vb}, {u}, {kind}, {mode}>",
                                f"{_A32 if vb == 32 else _A16}; {modes[mode]}; {knob}", DISPATCH))
    return tuple(out)


LEDGER = {
    # ---- amax.cu --------------------------------------------------------------------------------------------------
    "amax_tensor_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_per_tensor",),
        "variants": tuple((f"b200q::amax_tensor_kernel<{{T}}, {vb}, {u}>",
                           f"{'vec_bytes unset' if vb == 32 else 'vec_bytes=16'}; "
                           f"{'amax_unroll unset' if u == 4 else f'amax_unroll={u}'} (misalignment: scalar head)",
                           DISPATCH) for vb in (32, 16) for u in (1, 2, 4, 8)),
    },
    "amax_tensor_multi_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_per_tensor_multi",),
        "variants": (("b200q::amax_tensor_multi_kernel<{T}, 32, 4>", "always", KERNELS_T),),
    },
    "amax_tensor_tma_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_per_tensor",),
        "variants": (("b200q::amax_tensor_tma_kernel<{T}>", "amax_tma=1", KERNELS_T),),
    },
    "amax_rows_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_rows",),
        "variants": tuple((f"b200q::amax_rows_kernel<{{T}}, {vb}, {ln}>",
                           f"{'x 32-byte aligned, 32-byte rows' if vb == 32 else 'x 16-byte aligned, 16-byte rows'}; "
                           f"{ln // 2 + 1}..{ln if ln < 32 else 255} vectors per row", DISPATCH)
                          for vb in (32, 16) for ln in (2, 4, 8, 16, 32)),
    },
    "amax_longrows_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_rows",),
        "variants": tuple((f"b200q::amax_longrows_kernel<{{T}}, {vb}>", f"{vb}-byte vectors; >= 256 vectors per row",
                           DISPATCH) for vb in (32, 16)),
    },
    "amax_vecrows_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_rows",),
        "variants": tuple((f"b200q::amax_vecrows_kernel<{{T}}, {vb}>", f"{vb}-byte vectors; rows of one vector",
                           DISPATCH) for vb in (32, 16)),
    },
    "amax_rows_scalar_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_rows",),
        "variants": (("b200q::amax_rows_scalar_kernel<{T}>", "x or the row not 16-byte aligned", DISPATCH),),
    },
    "cols_reduce_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_cols", "b200q_abssum_cols"),
        "variants": tuple((f"b200q::cols_reduce_kernel<{{T}}, {vb}, {m}>",
                           ("x 32-byte aligned, 32-byte rows, n_cols >= 2048" if vb == 32 else
                            "x 16-byte aligned, 16-byte rows, n_cols < 2048 or 16-byte aligned")
                           + ("; amax" if m == 0 else "; abs sum"), DISPATCH) for vb in (32, 16) for m in (0, 1)),
    },
    "cols_reduce_scalar_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_cols", "b200q_abssum_cols"),
        "variants": tuple((f"b200q::cols_reduce_scalar_kernel<{{T}}, {m}>", "x or the row not 16-byte aligned",
                           DISPATCH) for m in (0, 1)),
    },
    "amax_export_kernel": {
        "file": "amax.cu", "entry": ("b200q_amax_export",),
        "variants": (("b200q::amax_export_kernel", "always", KERNELS_T),),
    },
    # ---- fake_quant.cu --------------------------------------------------------------------------------------------
    "fake_quant_kernel": {
        "file": "fake_quant.cu", "entry": ("b200q_fake_quant_int", "b200q_fake_quant_fp8", "b200q_fake_quant_fp8_eager"),
        "variants": _fq_variants(),
    },
    "fake_quant_scalar_kernel": {
        "file": "fake_quant.cu", "entry": ("b200q_fake_quant_int", "b200q_fake_quant_fp8", "b200q_fake_quant_fp8_eager"),
        "variants": tuple((f"b200q::fake_quant_scalar_kernel<{{T}}, {k}>",
                           "x or y not 16-byte aligned, or the elements past the last whole vector", DISPATCH)
                          for k in (0, 1, 2)),
    },
    # ---- nvfp4.cu -------------------------------------------------------------------------------------------------
    "nvfp4_dyn_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_fake_quant_nvfp4",),
        "variants": tuple((f"b200q::nvfp4_dyn_kernel<{{T}}, {vb}, {u}>",
                           f"row_len % 16 == 0; {_A32 if vb == 32 else _A16}; "
                           f"{'nvfp4_unroll unset' if u == 2 else f'nvfp4_unroll={u}'}", DISPATCH)
                          for vb in (32, 16) for u in (1, 2, 4)),
    },
    "nvfp4_dyn_tma_store_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_fake_quant_nvfp4",),
        "variants": (("b200q::nvfp4_dyn_tma_store_kernel<{T}, 2>", "nvfp4_tma_store=1, 32-byte aligned, whole tiles",
                      KERNELS_T),),
    },
    "nvfp4_dyn_multi_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_fake_quant_nvfp4_multi", "b200q_collect_fake_quant_nvfp4_multi"),
        "variants": (("b200q::nvfp4_dyn_multi_kernel<{T}, 32, 2, false>", "fake quant of a table", KERNELS_T),
                     ("b200q::nvfp4_dyn_multi_kernel<{T}, 32, 2, true>", "fused collect + fake quant", FUSED_T)),
    },
    "nvfp4_dyn_multi_fixup_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_fake_quant_nvfp4_multi_fixup",),
        "variants": (("b200q::nvfp4_dyn_multi_fixup_kernel<{T}, 32, 2>", "always", STORE_T),),
    },
    "nvfp4_dyn_ragged_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_fake_quant_nvfp4",),
        "variants": (("b200q::nvfp4_dyn_ragged_kernel<{T}>", "row_len % 16 != 0, or x / y not 16-byte aligned",
                      DISPATCH),),
    },
    "nvfp4_static_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_fake_quant_nvfp4_static",),
        "variants": tuple((f"b200q::nvfp4_static_kernel<{{T}}, {vb}, {u}>",
                           f"{_A32 if vb == 32 else _A16}; {'nvfp4_unroll unset' if u == 2 else f'nvfp4_unroll={u}'}",
                           DISPATCH) for vb in (32, 16) for u in (1, 2, 4)),
    },
    "nvfp4_pack_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_pack_nvfp4", "b200q_pack_nvfp4_scale2", "b200q_pack_nvfp4_static"),
        "variants": tuple((f"b200q::nvfp4_pack_kernel<{{T}}, {vb}, {s}, {u}>",
                           f"x {vb}-byte aligned; {'static' if s == 'true' else 'dynamic'}; "
                           f"{'pack_unroll unset' if u == 2 else 'pack_unroll=1'}", DISPATCH)
                          for vb in (32, 16) for s in _B for u in (1, 2)),
    },
    "nvfp4_unpack_kernel": {
        "file": "nvfp4.cu", "entry": ("b200q_unpack_nvfp4",),
        "variants": (("b200q::nvfp4_unpack_kernel<{T}>", "always", DISPATCH),),
    },
    # ---- pack.cu --------------------------------------------------------------------------------------------------
    "int4_pack_kernel": {
        "file": "pack.cu", "entry": ("b200q_pack_int4_blockwise",),
        "variants": tuple((f"b200q::int4_pack_kernel<{{T}}, {vb}, {ln}>",
                           f"block_size {16 * ln}; x {vb}-byte aligned", DISPATCH) for vb in (32, 16) for ln in _L),
    },
    "int4_pack_generic_kernel": {
        "file": "pack.cu", "entry": ("b200q_pack_int4_blockwise",),
        "variants": (("b200q::int4_pack_generic_kernel<{T}>",
                      "block_size not 16 * 2^k, or x not 16-byte aligned", DISPATCH),),
    },
    "int4_unpack_kernel": {
        "file": "pack.cu", "entry": ("b200q_unpack_int4_blockwise",),
        "variants": (("b200q::int4_unpack_kernel<{T}>", "always", DISPATCH),),
    },
    "int4_export_kernel": {
        "file": "pack.cu", "entry": ("b200q_pack_int4_export",),
        "variants": (("b200q::int4_export_kernel<{T}, 0>", "the scale dtype differs from w's, or fp32", DISPATCH),
                     ("b200q::int4_export_kernel<b200q::BF16Tag, 1>", "bf16 w and scale", DISPATCH),
                     ("b200q::int4_export_kernel<b200q::F16Tag, 2>", "fp16 w and scale", DISPATCH)),
    },
    "fp8_pack_kernel": {
        "file": "pack.cu", "entry": ("b200q_pack_fp8", "b200q_pack_int8"),
        "variants": tuple((f"b200q::fp8_pack_kernel<{{T}}, {vb}, {r}, {i}>",
                           f"x {vb}-byte aligned, q 4-byte aligned; quotient "
                           f"{'rounded to x dtype' if r == 'true' else 'kept in fp32'}; {'INT8' if i == 'true' else 'FP8'}",
                           DISPATCH) for vb in (32, 16) for r in _B for i in _B),
    },
    "fp8_pack_scalar_kernel": {
        "file": "pack.cu", "entry": ("b200q_pack_fp8", "b200q_pack_int8"),
        "variants": tuple((f"b200q::fp8_pack_scalar_kernel<{{T}}, {r}, {i}>",
                           "x not 16-byte aligned, q % 4 != 0, or the elements past the last whole vector", DISPATCH)
                          for r in _B for i in _B),
    },
    "fp8_unpack_kernel": {
        "file": "pack.cu", "entry": ("b200q_unpack_fp8", "b200q_unpack_int8"),
        "variants": tuple((f"b200q::fp8_unpack_kernel<{{T}}, {i}>", "INT8" if i == "true" else "FP8", DISPATCH)
                          for i in _B),
    },
    # ---- mx.cu ----------------------------------------------------------------------------------------------------
    "mx_fq_kernel": {
        "file": "mx.cu", "entry": ("b200q_fake_quant_mx",),
        "variants": (("b200q::mx_fq_kernel<{T}, 2, *>", "block 32, row_len % 32 == 0, x and y 32-byte aligned", DISPATCH),
                     ("b200q::mx_fq_kernel<{T}, 1, *>", "block 16, row_len % 16 == 0, x and y 32-byte aligned", DISPATCH)),
    },
    "mx_fq_generic_kernel": {
        "file": "mx.cu", "entry": ("b200q_fake_quant_mx",),
        "variants": (("b200q::mx_fq_generic_kernel<{T}, *>", "block 8, a ragged row, or x / y not 32-byte aligned",
                      DISPATCH),),
    },
    "mxfp8_pack_kernel": {
        "file": "mx.cu", "entry": ("b200q_pack_mxfp8",),
        "variants": (("b200q::mxfp8_pack_kernel<{T}>", "both the aligned and the element-wise branch", DISPATCH),),
    },
    "mxfp8_unpack_kernel": {
        "file": "mx.cu", "entry": ("b200q_unpack_mxfp8",),
        "variants": (("b200q::mxfp8_unpack_kernel<{T}>", "both the aligned and the element-wise branch", DISPATCH),),
    },
    "mxfp4_pack_kernel": {
        "file": "mx.cu", "entry": ("b200q_pack_mxfp4",),
        "variants": (("b200q::mxfp4_pack_kernel<{T}>", "both the aligned (block 32) and the element-wise branch",
                      DISPATCH),),
    },
    "mxfp4_unpack_kernel": {
        "file": "mx.cu", "entry": ("b200q_unpack_mxfp4",),
        "variants": (("b200q::mxfp4_unpack_kernel<{T}>", "both the aligned (block 32) and the element-wise branch",
                      DISPATCH),),
    },
    # ---- nf4.cu ---------------------------------------------------------------------------------------------------
    "nf4_pack_kernel": {
        "file": "nf4.cu", "entry": ("b200q_pack_nf4",),
        "variants": tuple((f"b200q::nf4_pack_kernel<{{T}}, 32, {ln}>",
                           f"block_size {16 * ln}, x 32-byte aligned; fp32, or nf4_lut=2", DISPATCH) for ln in _L),
    },
    "nf4_lut_init_kernel": {
        "file": "nf4.cu", "entry": ("b200q_pack_nf4",),
        "variants": (("b200q::nf4_lut_init_kernel<{T}>", "first LUT pack of a 16-bit dtype on a device", DISPATCH),),
    },
    "nf4_pack_lut_kernel": {
        "file": "nf4.cu", "entry": ("b200q_pack_nf4",),
        "variants": tuple((f"b200q::nf4_pack_lut_kernel<{{T}}, {ln}>",
                           f"block_size {16 * ln}, x 32-byte aligned, bf16 / fp16, nf4_lut unset", DISPATCH)
                          for ln in _L),
    },
    "nf4_pack_generic_kernel": {
        "file": "nf4.cu", "entry": ("b200q_pack_nf4",),
        "variants": (("b200q::nf4_pack_generic_kernel<{T}>", "block_size not 16 * 2^k, or x not 32-byte aligned",
                      DISPATCH),),
    },
    "nf4_unpack_kernel": {
        "file": "nf4.cu", "entry": ("b200q_unpack_nf4",),
        "variants": (("b200q::nf4_unpack_kernel<{T}>", "the scales' dtype; aligned and element-wise branch", DISPATCH),),
    },
    # ---- bias.cu --------------------------------------------------------------------------------------------------
    "reduce_keep_kernel": {
        "file": "bias.cu", "entry": ("b200q_reduce_keep",),
        "variants": (("b200q::reduce_keep_kernel<{T}>", "n_cols a whole number of 16-byte vectors, x 16-byte aligned",
                      DISPATCH),),
    },
    "reduce_keep_generic_kernel": {
        "file": "bias.cu", "entry": ("b200q_reduce_keep",),
        "variants": (("b200q::reduce_keep_generic_kernel<{T}>", "ragged n_cols or x not 16-byte aligned", DISPATCH),),
    },
    # ---- histogram.cu ---------------------------------------------------------------------------------------------
    "hist_plan_kernel": {
        "file": "histogram.cu", "entry": ("b200q_hist_plan",),
        "variants": (("b200q::hist_plan_kernel", "always", CALIB_T),),
    },
    "histogram_kernel": {
        "file": "histogram.cu", "entry": ("b200q_histogram", "b200q_histogram_ex", "b200q_histogram_planned"),
        "variants": (("b200q::histogram_kernel<{T}, 16, false, 512>", "no scratch (or fp32, or hist_variant=2)",
                      DISPATCH),
                     ("b200q::histogram_kernel<{T}, 16, true, 1024>", "hist_variant=1", DISPATCH)),
    },
    "hist_pattern_count_kernel": {
        "file": "histogram.cu", "entry": ("b200q_histogram_ex",),
        "variants": (("b200q::hist_pattern_count_kernel<{T}>", "16-bit x with scratch: fp16, or bf16 with hist_hot=2",
                      DISPATCH),),
    },
    "hist_pattern_hot_kernel": {
        "file": "histogram.cu", "entry": ("b200q_histogram_ex",),
        "variants": (("b200q::hist_pattern_hot_kernel", "bf16 x with scratch, hist_hot unset", DISPATCH),),
    },
    "hist_pattern_bin_kernel": {
        "file": "histogram.cu", "entry": ("b200q_histogram_ex",),
        "variants": (("b200q::hist_pattern_bin_kernel<{T}>", "16-bit x with scratch", DISPATCH),),
    },
    "block_log2_hist_kernel": {
        "file": "histogram.cu", "entry": ("b200q_nvfp4_block_log2_hist",),
        "variants": tuple((f"b200q::block_log2_hist_kernel<{{T}}, {vb}>", f"x {vb}-byte aligned", DISPATCH)
                          for vb in (32, 16)),
    },
    # ---- hist_search.cu -------------------------------------------------------------------------------------------
    "hist_percentile_kernel": {
        "file": "hist_search.cu", "entry": ("b200q_hist_search_percentile",),
        "variants": (("b200q::hist_percentile_kernel", "always", CALIB_T),),
    },
    "hist_prefix_kernel": {
        "file": "hist_search.cu", "entry": ("b200q_hist_search_entropy",),
        "variants": (("b200q::hist_prefix_kernel", "always", CALIB_T),),
    },
    "hist_entropy_kernel": {
        "file": "hist_search.cu", "entry": ("b200q_hist_search_entropy",),
        "variants": (("b200q::hist_entropy_kernel", "always", CALIB_T),),
    },
    "hist_mse_kernel": {
        "file": "hist_search.cu", "entry": ("b200q_hist_search_mse",),
        "variants": (("b200q::hist_mse_kernel", "always", CALIB_T),),
    },
    # ---- search.cu ------------------------------------------------------------------------------------------------
    "scale_cols_kernel": {
        "file": "search.cu", "entry": ("b200q_scale_cols",),
        "variants": (("b200q::scale_cols_kernel<{T}, 16>", "x and y 16-byte aligned, whole vectors per row", DISPATCH),),
    },
    "scale_cols_scalar_kernel": {
        "file": "search.cu", "entry": ("b200q_scale_cols",),
        "variants": (("b200q::scale_cols_scalar_kernel<{T}>", "x or y not 16-byte aligned, or ragged rows", DISPATCH),),
    },
    "awq_scale_fq_kernel": {
        "file": "search.cu", "entry": ("b200q_awq_scale_fake_quant",),
        "variants": tuple((f"b200q::awq_scale_fq_kernel<{{T}}, {vb}, {ln}, {vs}>",
                           f"block_size {16 * ln}; " + (
                               "16-bit w, scale of w's dtype, w / y / scale 32-byte aligned" if vs == "true" else
                               "w and y 32-byte aligned, fp32 w or another scale dtype" if vb == 32 else
                               "w or y 16- but not 32-byte aligned"), DISPATCH)
                          for vb, vs in ((32, "true"), (32, "false"), (16, "false")) for ln in _L),
    },
    "awq_weight_scale_kernel": {
        "file": "search.cu", "entry": ("b200q_awq_weight_scale_sums",),
        "variants": tuple((f"b200q::awq_weight_scale_kernel<{{T}}, {vb}, {ln}>",
                           f"block_size {16 * ln}; w {vb}-byte aligned with {vb}-byte rows", DISPATCH)
                          for vb in (32, 16) for ln in _L),
    },
    "mse_sweep_rows_kernel": {
        "file": "search.cu", "entry": ("b200q_mse_sweep_rows",),
        "variants": (("b200q::mse_sweep_rows_kernel<{T}>", "always", DISPATCH),),
    },
    "mse_sweep_kernel": {
        "file": "search.cu", "entry": ("b200q_mse_sweep",),
        "variants": (("b200q::mse_sweep_kernel<{T}, 16>", "always", DISPATCH),),
    },
    "fp8_sweep_kernel": {
        "file": "search.cu", "entry": ("b200q_nvfp4_fp8_scale_sweep", "b200q_nvfp4_fp8_scale_sweep_ex"),
        "variants": tuple((f"b200q::fp8_sweep_kernel<{{T}}, {vb}>", f"w {vb}-byte aligned", DISPATCH)
                          for vb in (32, 16)),
    },
    "fp8_sweep_hessian_kernel": {
        "file": "search.cu", "entry": ("b200q_nvfp4_fp8_scale_sweep_hessian",),
        "variants": (("b200q::fp8_sweep_hessian_kernel<{T}>", "always", HESSIAN_T),),
    },
    "nvfp4_static_mse_sweep_kernel": {
        "file": "search.cu", "entry": ("b200q_nvfp4_static_mse_sweep",),
        "variants": tuple((f"b200q::nvfp4_static_mse_sweep_kernel<{{T}}, {vb}>", f"w {vb}-byte aligned", DISPATCH)
                          for vb in (32, 16)),
    },
    # ---- hadamard.cu, gptq.cu, runtime.cu: instantiations tested by their own suites -------------------------------
    "hadamard_kernel": {
        "file": "hadamard.cu", "entry": ("b200q_hadamard", "b200q_fake_quant_nvfp4_rotated"),
        "variants": (("b200q::hadamard_kernel<{T}, *, *, *>", "block size, vector path, fused NVFP4 / amax", ROTATE_T),),
    },
    "gptq_block_kernel": {
        "file": "gptq.cu", "entry": ("b200q_gptq_block",),
        "variants": (("b200q::gptq_block_kernel<*>", "the quantizer format", GPTQ_T),),
    },
    "fastdiv_selftest_kernel": {
        "file": "runtime.cu", "entry": ("b200q_selftest_fastdiv",),
        "variants": (("b200q::fastdiv_selftest_kernel", "always", KERNELS_T),),
    },
    "e2m1_round_selftest_kernel": {
        "file": "runtime.cu", "entry": ("b200q_selftest_e2m1_round",),
        "variants": (("b200q::e2m1_round_selftest_kernel", "always", E2M1_T),),
    },
}

_TAG = r"b200q::(?:BF16|F16|F32)Tag"


def variant_regex(name: str) -> "re.Pattern":
    """The ledger name as a pattern over ``canonical`` kernel names."""
    parts = []
    for tok in re.split(r"(\{T\}|\*)", name):
        parts.append(_TAG if tok == "{T}" else r"[^<>]+?" if tok == "*" else re.escape(tok))
    return re.compile("^" + "".join(parts) + "$")


def canonical(demangled: str) -> str:
    """A demangled kernel name as the ledger spells it: no return type, no argument list, template arguments as
    ``int`` literals and ``true`` / ``false`` (demanglers differ: ``(int)16`` and ``(bool)1`` become ``16`` and
    ``true``)."""
    s = demangled.strip()
    s = re.sub(r"\(bool\)1\b", "true", re.sub(r"\(bool\)0\b", "false", s))
    s = re.sub(r"\((?:int|unsigned int|unsigned|long|unsigned long)\)(-?\d+)", r"\1", s)
    if s.startswith("void "):
        s = s[5:]
    depth = 0
    for i, c in enumerate(s):
        if c == "<":
            depth += 1
        elif c == ">":
            depth -= 1
        elif c == "(" and depth == 0:
            return s[:i].strip()
    return s


def variants_for(test: str):
    """``(kernel, name)`` of every ledger variant whose covering test is the module ``test``."""
    return [(k, v[0]) for k, e in LEDGER.items() for v in e["variants"] if v[2] == test]
