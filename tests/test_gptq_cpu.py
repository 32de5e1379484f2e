"""GPTQ host logic without a GPU: update_hessian and compute_hessian_inverse (the reference's known answers, and
against tests/golden/ref_gptq.npz: several batches, a dead column, the non-positive-definite fallback), the C oracle of
the GPTQ block (tools/gptq_oracle.c) bit for bit against the reference's gptq_blockwise_update run on CPU
(tools/gen_gptq_golden.py), the two rounding modes of the in-block update, the config validation, dispatch and the
layerwise refusal."""

import warnings

import numpy as np
import pytest
import torch

from oracle import golden
from tools import gptq_oracle as orc


@pytest.fixture(scope="module")
def ref():
    return golden.load("ref_gptq")


def _bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


def test_hessian_and_inverse_vs_reference(ref):
    from model_optimizer_b200.model_calib import compute_hessian_inverse, update_hessian

    h, n = torch.zeros(32, 32), 0
    for i in range(3):
        h, n = update_hessian(torch.from_numpy(ref[f"hess/x{i}"]), h, n)
    assert n == int(ref["hess/n3"])
    torch.testing.assert_close(h, torch.from_numpy(ref["hess/h3"]), rtol=1e-6, atol=1e-7)
    x = torch.from_numpy(np.concatenate([ref[f"hess/x{i}"].reshape(-1, 32) for i in range(3)]))
    h1, n1 = update_hessian(x, torch.zeros(32, 32), 0)
    assert n1 == int(ref["hess/n1"])
    torch.testing.assert_close(h1, torch.from_numpy(ref["hess/h1"]), rtol=1e-6, atol=1e-7)
    u = compute_hessian_inverse(torch.from_numpy(ref["hinv/h"]), torch.from_numpy(ref["hinv/w"]), 0.01)
    torch.testing.assert_close(u, torch.from_numpy(ref["hinv/u"]), rtol=1e-5, atol=1e-6)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        bad = compute_hessian_inverse(-torch.eye(8), torch.ones(4, 8), 0.01)
    assert torch.equal(bad, torch.from_numpy(ref["hinv/u_bad"]))


_FIXTURE_FORMATS = {
    "int8_row": lambda amax, nb: {"fmt": orc.FMT_INT, "amax": amax, "amax_row_stride": 1, "num_bits": 8},
    "fp8": lambda amax, nb: {"fmt": orc.FMT_FP8_EAGER, "amax": amax},
    "int4_b128": lambda amax, nb: {"fmt": orc.FMT_INT, "amax": amax, "amax_row_stride": nb // 128,
                                   "amax_col_block": 128, "num_bits": 4},
    "nvfp4_static": lambda amax, nb: {"fmt": orc.FMT_NVFP4_STATIC, "amax": amax, "amax_row_stride": nb // 16,
                                      "amax_col_block": 16},
    "nvfp4_dynamic": lambda amax, nb: {"fmt": orc.FMT_NVFP4_DYNAMIC, "amax": amax},
}


@pytest.mark.parametrize("nb,sdt,fname", [(nb, sdt, f) for nb in (16, 64, 128) for sdt in ("f32", "bf16")
                                           for f in _FIXTURE_FORMATS if f != "int4_b128" or nb == 128])
def test_oracle_block_vs_reference_bit_for_bit(ref, nb, sdt, fname):
    """The oracle in its fused-multiply-add mode (ATen's CPU addr_) equals the reference's gptq_blockwise_update."""
    key = f"block/{nb}/{sdt}"
    kw = _FIXTURE_FORMATS[fname](ref[f"{key}/{fname}/amax"], nb)
    if f"{key}/{fname}/global_amax" in ref:
        kw["global_amax"] = float(ref[f"{key}/{fname}/global_amax"])
    got, _ = orc.gptq_block(ref[f"{key}/w"], ref[f"{key}/u"], fma=True, **kw)
    want = ref[f"{key}/{fname}/out"]
    assert _bits_equal(got, want), int((got.view(np.uint32) != want.view(np.uint32)).sum())
    assert not _bits_equal(got, ref[f"{key}/w"])


def test_update_hessian_known_answers():
    from model_optimizer_b200.model_calib import update_hessian

    h, n = update_hessian(torch.ones(4, 8), torch.zeros(8, 8), 0)
    assert n == 4
    torch.testing.assert_close(h, torch.full((8, 8), 2.0))
    x = torch.randn(3, 5, 16, generator=torch.Generator().manual_seed(0))
    h3, n3 = torch.zeros(16, 16), 0
    for b in x:
        h3, n3 = update_hessian(b, h3, n3)
    h1, n1 = update_hessian(x, torch.zeros(16, 16), 0)
    assert n3 == n1 == 15
    torch.testing.assert_close(h3, h1, rtol=1e-5, atol=1e-6)
    h0 = torch.randn(16, 16)
    out, n0 = update_hessian(torch.zeros(0, 16), h0, 7)
    assert out is h0 and n0 == 7


def test_compute_hessian_inverse_dead_column_and_fallback():
    from model_optimizer_b200.model_calib import compute_hessian_inverse

    g = torch.Generator().manual_seed(1)
    x = torch.randn(64, 16, generator=g)
    h = 2 * x.T @ x / 64
    w = torch.randn(8, 16, generator=g)
    w[:, 5] = 0
    u = compute_hessian_inverse(h, w, 0.01)
    hd = h.clone()
    hd[5, :] = 0
    hd[:, 5] = 0
    hd[5, 5] = 1
    hd += 0.01 * torch.mean(torch.diag(hd)) * torch.eye(16)
    torch.testing.assert_close(u.T @ u, torch.linalg.inv(hd), rtol=1e-3, atol=1e-4)
    assert torch.equal(u, torch.triu(u))
    assert (u[5, 6:] == 0).all() and (u[:5, 5] == 0).all() and u[5, 5] > 0   # the dead column is decoupled
    bad = -torch.eye(16)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        out = compute_hessian_inverse(bad, torch.ones(4, 16), 0.01)
    assert torch.equal(out, torch.eye(16)) and any("positive definite" in str(r.message) for r in rec)


def _numpy_int8_block(w, u, amax, fma):
    """The recurrence restated with numpy float32 scalars (INT8 per tensor, narrow_range False)."""
    f = np.float32
    w = w.astype(np.float32).copy()
    rows, nb = w.shape
    q_out = np.zeros_like(w)
    e = np.zeros_like(w)
    scale = f(127) / f(amax)
    for r in range(rows):
        wk = w[r].copy()
        for i in range(nb):
            o = np.clip(np.rint(f(wk[i] * scale)), f(-128), f(127)).astype(np.float32)
            q = f(o / scale)
            err = f(f(wk[i] - q) / u[i, i])
            q_out[r, i], e[r, i] = q, err
            for j in range(i, nb):
                if fma:   # one rounding of the exact -err * u + w (float64 holds the product exactly)
                    wk[j] = f(np.float64(-err) * np.float64(u[i, j]) + np.float64(wk[j]))
                else:
                    wk[j] = f(wk[j] + f(-err * u[i, j]))
    return q_out, e


@pytest.mark.parametrize("fma", [False, True])
def test_oracle_recurrence_int8(fma):
    g = np.random.default_rng(3)
    w = (g.standard_normal((5, 16)) * 0.05).astype(np.float32)
    x = g.standard_normal((64, 16))
    h = x.T @ x / 64 + 0.01 * np.eye(16)
    u = np.linalg.cholesky(np.linalg.inv(h)).T.astype(np.float32)
    amax = np.float32(0.11)
    got_w, got_e = orc.gptq_block(w, u, orc.FMT_INT, [amax], fma=fma)
    want_w, want_e = _numpy_int8_block(w, u, amax, fma)
    # the float64 route of the fused product is exact except for double-rounding corner cases: compare closely
    np.testing.assert_allclose(got_w, want_w, rtol=0, atol=1e-7)
    np.testing.assert_allclose(got_e, want_e, rtol=1e-6, atol=1e-9)


def test_oracle_identity_u_is_plain_quant_and_modes_differ():
    g = np.random.default_rng(5)
    w = (g.standard_normal((32, 64)) * 0.05).astype(np.float32)
    qw, e = orc.gptq_block(w, np.eye(64, dtype=np.float32), orc.FMT_INT, [0.1])
    scale = np.float32(127) / np.float32(0.1)
    plain = (np.clip(np.rint(w * scale), -128, 127).astype(np.float32) / scale).astype(np.float32)
    assert np.array_equal(qw.view(np.uint32), plain.view(np.uint32))
    np.testing.assert_array_equal(e, (w - qw).astype(np.float32))
    # with a full factor the two roundings of the update (rounded product + add, one fused multiply-add) differ in E
    x = g.standard_normal((256, 64))
    u = np.linalg.cholesky(np.linalg.inv(x.T @ x / 256 + 0.01 * np.eye(64))).T.astype(np.float32)
    _, e_mul = orc.gptq_block(w, u, orc.FMT_NVFP4_DYNAMIC, [0.2], fma=False)
    _, e_fma = orc.gptq_block(w, u, orc.FMT_NVFP4_DYNAMIC, [0.2], fma=True)
    assert np.isfinite(e_mul).all() and np.isfinite(e_fma).all()
    assert not _bits_equal(e_mul, e_fma)
    np.testing.assert_allclose(e_mul, e_fma, rtol=1e-2, atol=1e-4)   # the same recurrence up to rounding


def test_config_validation_and_dispatch():
    from model_optimizer_b200 import model_calib
    from model_optimizer_b200.config import GPTQCalibConfig
    from model_optimizer_b200.model_quant import calibrate

    assert GPTQCalibConfig().perc_damp == 0.01 and GPTQCalibConfig().block_size == 128
    for bad in (0.0, -0.1, 1.5, True, "x"):
        with pytest.raises(ValueError):
            GPTQCalibConfig(perc_damp=bad)
    GPTQCalibConfig(perc_damp=1.0)
    for bad in (0, -4, 1.5, True):
        with pytest.raises(ValueError):
            GPTQCalibConfig(block_size=bad)
    with pytest.raises(ValueError):
        GPTQCalibConfig(method="awq")
    assert GPTQCalibConfig(layerwise={"enable": True}).layerwise_enabled
    assert not GPTQCalibConfig(layerwise=False).layerwise_enabled
    model = torch.nn.Linear(16, 8)
    with pytest.raises(NotImplementedError, match="backend.install"):
        calibrate(model, {"method": "gptq", "layerwise": {"enable": True}}, lambda m: None)
    with pytest.raises(ValueError, match="perc_damp"):
        calibrate(model, {"method": "gptq", "perc_damp": 2.0}, lambda m: None)
    assert model_calib.gptq.__name__ == "gptq"


def test_quantizer_desc_needs_calibrated_cuda_state():
    from model_optimizer_b200 import ops
    from model_optimizer_b200.config import QuantizerAttributeConfig
    from model_optimizer_b200.nn import TensorQuantizer

    q = TensorQuantizer(QuantizerAttributeConfig(num_bits=8, axis=0))
    assert ops.gptq_quantizer_desc(q, (8, 16)) is None             # no amax
    q.amax = torch.ones(8, 1)
    assert ops.gptq_quantizer_desc(q, (8, 16)) is None             # CPU state: the composed loop
