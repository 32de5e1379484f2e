"""Input rotation without a GPU: config forms and validation, the quantizer's rotate properties and forward ordering
(with a stand-in transform), the block choice and errors of normalized_hadamard_transform against the reference's
(tests/golden/ref_rotate.npz), the numpy oracle against the fp64 Hadamard product, the sharing signature, the drop-in
rebind and the C-ABI entry points."""

import ctypes

import numpy as np
import pytest
import torch

from model_optimizer_b200.config import QuantizerAttributeConfig, RotateConfig
from model_optimizer_b200.nn import functional as F
from model_optimizer_b200.nn import shared_input
from model_optimizer_b200.nn import tensor_quantizer as tq_mod
from model_optimizer_b200.nn.tensor_quantizer import TensorQuantizer
from oracle import golden
from tools.hadamard_oracle import hadamard, hadamard_f64, round_to


@pytest.fixture(scope="module")
def ref():
    return golden.load("ref_rotate")


# ---- config -----------------------------------------------------------------------------------------------------
def test_rotate_config_forms():
    assert QuantizerAttributeConfig().rotate is False
    assert QuantizerAttributeConfig(rotate=True).rotate is True
    c = QuantizerAttributeConfig(rotate={"enable": True, "mode": "rotate_back", "block_size": 128})
    assert c.rotate == RotateConfig(enable=True, mode="rotate_back", block_size=128)
    r = RotateConfig(enable=True, rotate_fp32=True)
    assert QuantizerAttributeConfig(rotate=r).rotate is r


@pytest.mark.parametrize("bad", [True, False, 0, -8, 1.5, "16"])
def test_rotate_block_size_validation(bad):
    with pytest.raises(ValueError, match="block_size must be a positive int"):
        RotateConfig(enable=True, block_size=bad)
    with pytest.raises(ValueError, match="block_size must be a positive int"):
        QuantizerAttributeConfig(rotate={"enable": True, "block_size": bad})


def test_rotate_mode_and_type_validation():
    with pytest.raises(ValueError, match="rotate mode"):
        RotateConfig(enable=True, mode="back")
    with pytest.raises(ValueError, match="rotate must be"):
        QuantizerAttributeConfig(rotate=1)


# ---- properties -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("form", ["bool", "dict", "config"])
def test_rotate_properties(form):
    full = {"enable": True, "mode": "rotate_back", "rotate_fp32": True, "block_size": 64}
    rot = {"bool": True, "dict": full, "config": RotateConfig(**full)}[form]
    q = TensorQuantizer(QuantizerAttributeConfig(rotate=rot))
    assert q.rotate_is_enabled is True
    if form == "bool":
        assert (q.rotate_back_is_enabled, q.rotate_is_fp32, q.rotate_block_size) == (False, False, None)
        assert q.extra_repr().endswith(" rotated")
    else:
        assert (q.rotate_back_is_enabled, q.rotate_is_fp32, q.rotate_block_size) == (True, True, 64)
        assert q.extra_repr().endswith(" rotated (rotate_back) (fp32) (block=64)")
    gen = q._state_gen
    q.disable_rotate()
    assert q._state_gen > gen
    assert type(q._rotate) is type(rot) if form != "dict" else isinstance(q._rotate, RotateConfig)
    assert (q.rotate_is_enabled, q.rotate_back_is_enabled, q.rotate_is_fp32, q.rotate_block_size) == (
        False, False, False, None)
    q.disable_rotate()                                   # idempotent
    assert not q.rotate_is_enabled


def test_checkpoint_dict_rotate_state():
    q = TensorQuantizer(QuantizerAttributeConfig())
    q._rotate = {"enable": True, "mode": "rotate_back", "block_size": 8}
    assert q.rotate_is_enabled and q.rotate_back_is_enabled and q.rotate_block_size == 8
    q.disable_rotate()
    assert q._rotate == {"enable": False, "mode": "rotate_back", "block_size": 8} and not q.rotate_is_enabled


def test_set_from_attribute_config_clears_rotation_and_bumps_state():
    q = TensorQuantizer(QuantizerAttributeConfig(rotate={"enable": True, "mode": "rotate_back", "block_size": 8}))
    gen = q._state_gen
    q.set_from_attribute_config({"enable": False})
    assert q._state_gen > gen and not q.rotate_is_enabled and not q.rotate_back_is_enabled


# ---- forward ordering (tensor_quantizer.py:1119-1221), with a stand-in transform --------------------------------------
def _stand_in(monkeypatch):
    calls = []

    def rotate_fn(inputs, rotate_fp32=False, block_size=None):
        calls.append((rotate_fp32, block_size))
        return inputs + 10

    monkeypatch.setattr(tq_mod, "normalized_hadamard_transform", rotate_fn)
    return calls


@pytest.mark.parametrize(("rotate", "expected_calls", "expected_fn"), [
    ({"enable": True}, [(False, None)], lambda x: (x + 10) * 2),
    ({"enable": True, "mode": "rotate_back", "rotate_fp32": True, "block_size": 8}, [(True, 8), (True, 8)],
     lambda x: ((x + 10) * 2) + 10),
])
def test_rotate_modes_order(monkeypatch, rotate, expected_calls, expected_fn):
    calls = _stand_in(monkeypatch)
    q = TensorQuantizer(QuantizerAttributeConfig(rotate=rotate))
    q._fake_quantize = lambda x: x * 2                     # the quantization step, as the reference test's backend
    x = torch.tensor([[1.0, 2.0]])
    assert torch.equal(q(x), expected_fn(x))
    assert calls == expected_calls


@pytest.mark.parametrize(("rotate", "n_calls", "expected_fn"), [
    ({"enable": True}, 1, lambda x: x + 10),
    ({"enable": True, "mode": "rotate_back"}, 2, lambda x: x + 20),
])
def test_disabled_rotate_roundtrip(monkeypatch, rotate, n_calls, expected_fn):
    calls = _stand_in(monkeypatch)
    x = torch.tensor([[1.0, 2.0]])
    q = TensorQuantizer(QuantizerAttributeConfig(rotate=rotate, enable=False))
    assert torch.equal(q(x), expected_fn(x)) and len(calls) == n_calls
    # enabled, but neither quantizing nor calibrating: the same rotated result
    calls.clear()
    q = TensorQuantizer(QuantizerAttributeConfig(rotate=rotate), if_quant=False, if_calib=False)
    assert torch.equal(q(x), expected_fn(x)) and len(calls) == n_calls


def test_rotate_back_rejects_real_quant_before_rotating(monkeypatch):
    def fail(inputs, rotate_fp32=False, block_size=None):
        raise AssertionError("rotate_back with fake_quant=False must fail before rotating")

    monkeypatch.setattr(tq_mod, "normalized_hadamard_transform", fail)
    q = TensorQuantizer(QuantizerAttributeConfig(num_bits=8, fake_quant=False,
                                                 rotate={"enable": True, "mode": "rotate_back"}))
    with pytest.raises(ValueError, match="rotate_back mode is only supported with fake_quant=True"):
        q(torch.tensor([[1.0, 2.0]]))


def test_no_rotation_leaves_forward_alone(monkeypatch):
    def fail(*a, **k):
        raise AssertionError("no rotation configured")

    monkeypatch.setattr(tq_mod, "normalized_hadamard_transform", fail)
    q = TensorQuantizer(QuantizerAttributeConfig(enable=False))
    x = torch.tensor([[1.0, 2.0]])
    assert q(x) is x


# ---- the wrapper's block choice and errors ------------------------------------------------------------------------
@pytest.mark.parametrize(("dim", "bs", "want"), [(64, None, 64), (96, None, 32), (1920, 128, 128), (1536, None, 512),
                                                 (16, 4, 4), (1, None, 1), (32768, None, 32768)])
def test_block_choice(dim, bs, want):
    assert F.rotate_block_size(dim, bs) == want


def test_wrapper_errors_match_reference(ref):
    for name, (dim, bs) in {"no_pow2_divisor": (7, None), "not_pow2": (96, 6), "not_divisible": (96, 64)}.items():
        with pytest.raises(Exception) as e:
            F.rotate_block_size(dim, bs)
        assert type(e.value).__name__ == str(ref[f"err/{name}/type"])
        assert str(e.value) == str(ref[f"err/{name}/msg"])


def test_wrapper_raises_on_cpu_and_above_32768():
    with pytest.raises(RuntimeError, match="CUDA"):
        F.normalized_hadamard_transform(torch.zeros(2, 64))
    with pytest.raises(ValueError, match="32768"):
        F.normalized_hadamard_transform(torch.zeros(1, 65536))


def test_reference_wrapper_outputs_are_the_oracle(ref):
    """The fixture's wrapper outputs (reference code around the stand-in) are the oracle of the chosen block, and
    rotate_fp32 did not change a bit."""
    for name, bs in (("d64", 64), ("d96", 32), ("d1920_b128", 128), ("d1536", 512), ("d16_b4", 4)):
        for d in ("bf16", "f16", "f32"):
            x = ref[f"wrap/{name}/{d}/fp32=0/x"]
            y0, y1 = ref[f"wrap/{name}/{d}/fp32=0/y"], ref[f"wrap/{name}/{d}/fp32=1/y"]
            assert np.array_equal(y0.view(np.uint32), hadamard(x, bs, d).view(np.uint32)), (name, d)
            assert np.array_equal(y0.view(np.uint32), y1.view(np.uint32)), (name, d)


# ---- the oracle ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", range(0, 13))
def test_oracle_vs_fp64_product(k):
    b = 1 << k
    x = np.random.default_rng(k).standard_normal((3, 2 * b)).astype(np.float32)
    y = hadamard(x, b, "f32")
    exact = hadamard_f64(x, b)
    tol = (k + 1) * 2.0 ** -23 * np.abs(x.reshape(-1, b)).sum(axis=1).max() / np.sqrt(b) + 1e-30
    assert np.max(np.abs(y - exact)) <= tol
    back = hadamard(y, b, "f32")                          # an involution up to rounding
    assert np.max(np.abs(back - x)) <= 2 * tol + 4 * 2.0 ** -23 * np.abs(x).max()


def test_oracle_scale_and_specials():
    for k in range(0, 16, 2):                               # even k: the scale is an exact power of 2
        assert np.float32((1 << k) ** -0.5) == np.float32(2.0 ** (-k // 2))
    x = np.array([[np.inf, 1.0, 0.0, -0.0], [np.nan, 0, 0, 0], [0.0, -0.0, 0.0, -0.0]], np.float32)
    y = hadamard(x, 4, "bf16")
    assert np.isinf(y[0, 0]) and np.isnan(y[1]).all() and (y[2] == 0).all()
    assert np.array_equal(round_to(np.float32([1 + 2 ** -8]), "bf16"), np.float32([1.0]))  # tie to even


# ---- sharing signature, drop-in rebind, C-ABI -------------------------------------------------------------------------
def test_signature_separates_rotations():
    cfgs = [{}, {"rotate": True}, {"rotate": {"enable": True, "mode": "rotate_back"}},
            {"rotate": {"enable": True, "block_size": 32}}]
    sigs = [shared_input.signature(TensorQuantizer(QuantizerAttributeConfig(**c))) for c in cfgs]
    assert len(set(sigs)) == len(sigs)
    # fp32 vs default rotation give the same bits, so they may share
    a = TensorQuantizer(QuantizerAttributeConfig(rotate={"enable": True, "rotate_fp32": True}))
    assert shared_input.signature(a) == sigs[1]


def test_backend_rebinds_the_transform(monkeypatch):
    from baseline import ref_env

    if not ref_env.available():
        pytest.skip("the reference is not installed in baseline/_ref")
    ref_env.activate()
    from modelopt.torch.quantization.nn.modules import tensor_quantizer as ref_tq

    from model_optimizer_b200 import _lib, backend

    try:
        _lib.load()
    except _lib.B200QuantError:
        pytest.skip("the CUDA library is not built")
    host_calls = []

    def host_transform(inputs, rotate_fp32=False, block_size=None):   # the host application's own function
        host_calls.append((rotate_fp32, block_size))
        return inputs + 1

    monkeypatch.setattr(ref_tq, "normalized_hadamard_transform", host_transform)
    backend.install()
    try:
        assert ref_tq.normalized_hadamard_transform is not host_transform
        before = backend.stats["fn.normalized_hadamard_transform"]
        x = torch.zeros(2, 64)
        # CPU tensors are outside the engine's scope: handed back to the host's function, not counted
        assert torch.equal(ref_tq.normalized_hadamard_transform(x, True, 32), x + 1)
        assert host_calls == [(True, 32)]
        assert backend.stats["fn.normalized_hadamard_transform"] == before
    finally:
        backend.uninstall()
    assert ref_tq.normalized_hadamard_transform is host_transform


def test_cabi_rotation_symbols():
    import __graft_entry__ as g

    lib = ctypes.CDLL(g.build_cuda())
    for s in ("b200q_hadamard", "b200q_fake_quant_nvfp4_rotated"):
        assert hasattr(lib, s), s
    lib.b200q_hadamard.restype = ctypes.c_int
    lib.b200q_last_error.restype = ctypes.c_char_p
    # argument checks run before any device work
    for bs, msg in ((3, b"power of 2"), (65536, b"power of 2"), (32, b"multiple of block_size")):
        assert lib.b200q_hadamard(None, None, 2, ctypes.c_size_t(0), ctypes.c_size_t(16), ctypes.c_size_t(bs), None,
                                  None) == 1
        assert msg in lib.b200q_last_error()


def test_oracle_is_stage_ordered():
    """The oracle's stage order is the kernel's: a different order changes fp32 bits for some inputs, so the
    restatement is not order-free and a GPU bit-exact match pins the order."""
    rng = np.random.default_rng(3)
    x = (rng.standard_normal((64, 8)) * np.exp2(rng.integers(-20, 20, (64, 8)))).astype(np.float32)

    def reversed_order(v):
        v = v.copy()
        for h in (4, 2, 1):
            w = v.reshape(-1, 8 // (2 * h), 2, h)
            a, b = w[:, :, 0, :].copy(), w[:, :, 1, :].copy()
            w[:, :, 0, :], w[:, :, 1, :] = a + b, a - b
            v = w.reshape(-1, 8)
        return v * np.float32(8 ** -0.5)

    assert not np.array_equal(hadamard(x, 8, "f32"), reversed_order(x))
