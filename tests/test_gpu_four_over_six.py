"""Four-Over-Six and the static NVFP4 multiplier search on the GPU.

* ``b200q_nvfp4_static_mse_sweep`` against the numpy oracle (tools/nvfp4_mse_oracle.py, ATen's CUDA sum order), bit
  for bit in ``best_amax`` and in every loss: bf16 / fp16 / fp32, 1, 7 and 2^20 + 3 blocks, 1 / 2 / 39 / 128
  candidates, fp8_max_norm 448 and 256, all-zero blocks, NaN / inf, E4M3 block-scale underflow and saturation, and
  blocks on which the two Four-Over-Six candidates tie exactly or within one ulp;
* against the reference's loop composed with torch on the GPU (the engine's static fake quant in fp32,
  ``F.mse_loss``, ``torch.sum(dim=1)``, ``argmin``), and over the reference's own Triton static kernel where
  ``oracle/_ref`` was built;
* the mirror's ``quantize(model, NVFP4_FOUR_OVER_SIX_CFG)`` against the reference's CPU run
  (tests/golden/ref_four_over_six.npz), and the drop-in against stock ``mtq.quantize`` where the reference is installed.
"""

import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import golden
from tools import nvfp4_mse_oracle as mo

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TDT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
LINEARS = ("q_proj", "k_proj", "v_proj", "o_proj")
FOS = np.float32([1.0, 1.5])


@pytest.fixture(scope="module")
def ops():
    from model_optimizer_b200 import ops as _ops

    return _ops


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same(a, b):
    """bit-equal, any NaN counting as equal to any NaN."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    return bool(np.all((bits(a) == bits(b)) | (np.isnan(a) & np.isnan(b))))


def weight_blocks(n_blocks, dtype, seed):
    """Gaussian blocks with heavy tails, then the special cases at the front."""
    rng = np.random.default_rng(seed)
    w = rng.standard_normal((n_blocks, 16)).astype(np.float32)
    w *= np.exp(rng.standard_normal((n_blocks, 1)) * 2).astype(np.float32)
    specials = [np.zeros(16, np.float32),                                                  # all zero
                np.float32([6, 3] + [0] * 14),                                             # exact 4/6 tie (see below)
                np.float32([6, 0, 1.5, 0.75] + [0] * 12),
                np.where(np.arange(16) == 3, np.float32(np.nan), np.float32(1)),           # NaN
                np.where(np.arange(16) == 5, np.float32(np.inf), np.float32(-2)),          # inf
                np.full(16, 1e-30, np.float32),                                            # block scale underflows
                np.full(16, 3e37, np.float32)]                                             # scale saturates
    for i, s in enumerate(specials[:n_blocks]):
        w[i] = s
    return o_round(w, dtype)


def o_round(w, dtype):
    from oracle import oracle_np as o

    with np.errstate(over="ignore", invalid="ignore"):
        return o.round_to(w, dtype)


def block_amax(w):
    with np.errstate(invalid="ignore"):
        return np.max(np.abs(w), axis=1).astype(np.float32)


def run(ops, w, a0, g, mult, norm, dtype):
    wd = torch.from_numpy(w).cuda().to(TDT[dtype])
    loss = torch.empty(len(mult), w.shape[0], dtype=torch.float32, device="cuda")
    best = ops.nvfp4_static_mse_sweep(wd, torch.from_numpy(a0).cuda(), torch.tensor([g]).cuda(),
                                      torch.from_numpy(mult).cuda(), norm, loss_out=loss)
    return best.cpu().numpy(), loss.cpu().numpy()


@pytest.mark.parametrize("dtype", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("n_blocks", [1, 7, 4099])
@pytest.mark.parametrize("n_cand", [1, 2, 39, 128])
@pytest.mark.parametrize("norm", [448.0, 256.0])
def test_kernel_vs_oracle(ops, dtype, n_blocks, n_cand, norm):
    w = weight_blocks(n_blocks, dtype, seed=n_blocks * 7 + n_cand)
    a0 = block_amax(w)
    finite = a0[np.isfinite(a0)]
    g = np.float32(finite.max() if finite.size else 1.0)
    if norm == 256.0 and n_blocks >= 7:
        g = np.float32(6 * 256)        # block scale a/6 FP8-exact: the two 4/6 candidates tie on blocks 1 and 2
    mult = FOS if n_cand == 2 else np.linspace(0.25, 4.0, n_cand, dtype=np.float32)
    best, loss = run(ops, w, a0, g, mult, norm, dtype)
    want, _, wloss = mo.search(w, a0, g, mult, norm, "cuda")
    assert same(loss, wloss)
    assert same(best, want)
    if norm == 256.0 and n_blocks >= 7 and n_cand == 2:
        assert loss[0, 1] == loss[1, 1] == 0 and best[1] == a0[1]          # exact tie: the first candidate wins


@pytest.mark.parametrize("dtype", ["bf16", "f32"])
def test_kernel_vs_oracle_large(ops, dtype):
    """2^20 + 3 blocks, the Four-Over-Six pair at 256."""
    w = weight_blocks((1 << 20) + 3, dtype, seed=11)
    a0 = block_amax(w)
    g = np.float32(np.nanmax(np.where(np.isfinite(a0), a0, 0)))
    best, loss = run(ops, w, a0, g, FOS, 256.0, dtype)
    want, _, wloss = mo.search(w, a0, g, FOS, 256.0, "cuda")
    assert same(loss, wloss) and same(best, want)


def test_kernel_near_ties(ops):
    """Blocks on which the two 4/6 losses are equal or one ulp apart (picked from many random blocks by the
    oracle): the first-minimum rule and the sum order decide them."""
    w = weight_blocks(1 << 18, "bf16", seed=5)[7:]
    a0 = block_amax(w)
    g = np.float32(a0.max())
    _, _, l = mo.search(w, a0, g, FOS, 256.0, "cuda")
    d = np.abs(bits(l[0]).astype(np.int64) - bits(l[1]).astype(np.int64))
    pick = np.nonzero(d <= 1)[0]
    assert pick.size >= 8, pick.size
    best, loss = run(ops, np.ascontiguousarray(w[pick]), a0[pick], g, FOS, 256.0, "bf16")
    want, _, wloss = mo.search(w[pick], a0[pick], g, FOS, 256.0, "cuda")
    assert same(loss, wloss) and same(best, want)


def composed(ops, w, a0, g, mult, norm):
    """The reference's MseCalibrator loop (calib/mse.py:84-172) with torch on the GPU and the engine's static fake
    quant in fp32."""
    x = w.reshape(-1, 16).to(torch.float32)
    losses = []
    for m in mult:
        xq = ops.fake_quant_nvfp4_static(x, a0 * m, g, True, norm)
        losses.append(F.mse_loss(x, xq, reduction="none").sum(dim=1))
    return a0 * mult[torch.argmin(torch.stack(losses), dim=0)]


@pytest.mark.parametrize("dtype", ["bf16", "f16", "f32"])
@pytest.mark.parametrize("n_cand", [2, 39])
def test_kernel_vs_torch_composition(ops, dtype, n_cand):
    torch.manual_seed(0)
    w = (torch.randn(1024, 4096, device="cuda") * (1 + 8 * (torch.rand(1024, 4096, device="cuda") < 0.01))).to(TDT[dtype])
    a0 = w.reshape(-1, 16).abs().amax(dim=1).float()
    g = a0.max().reshape(1)
    norm = 256.0 if n_cand == 2 else 448.0
    mult = torch.linspace(1.0, 1.5, 2, device="cuda") if n_cand == 2 else torch.linspace(0.25, 4.0, 39, device="cuda")
    got = ops.nvfp4_static_mse_sweep(w, a0, g, mult, norm)
    want = composed(ops, w, a0, g, mult, norm)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))


def test_kernel_vs_reference_triton_composition(ops):
    """The same loop over the reference's own Triton static kernel at 256 (scales as compute_fp4_scales builds them
    on the GPU).  The Triton kernel's division rounds differently on a few exact E2M1 ties
    (test_gpu_vs_reference_triton.py), so the winners agree on all but a few blocks."""
    import importlib.machinery
    import importlib.util

    spec = importlib.util.spec_from_file_location(
        "_vs_reference_triton", os.path.join(ROOT, "tests", "test_gpu_vs_reference_triton.py"))
    vrt = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(vrt)
    REF, RefTritonKernel = vrt.REF, vrt.RefTritonKernel
    p = os.path.join(REF, "modelopt_cuda_ext_fp8.so")
    if not os.path.exists(p):
        pytest.skip("reference fp8 extension not built")
    loader = importlib.machinery.ExtensionFileLoader("modelopt_cuda_ext_fp8", p)
    ext8 = importlib.util.module_from_spec(importlib.util.spec_from_loader("modelopt_cuda_ext_fp8", loader))
    loader.exec_module(ext8)
    k = RefTritonKernel("fp4_static_f32")
    torch.manual_seed(1)
    w = torch.randn(512, 2048, device="cuda").to(torch.bfloat16)
    a0 = w.reshape(-1, 16).abs().amax(dim=1).float()
    g = a0.max()
    mult = torch.linspace(1.0, 1.5, 2, device="cuda")
    x = w.reshape(-1, 16).float().contiguous()
    losses = []
    for m in mult:
        amax = a0 * m
        scale = ext8.fake_e4m3fy(amax / 6.0, (g * (448.0 / 256.0) / 6.0).reshape(1))   # fp4_kernel.py:232-244
        y = torch.empty_like(x)
        k((amax.numel(),), x.data_ptr(), y.data_ptr(), scale.contiguous().data_ptr(), amax.numel())
        losses.append(F.mse_loss(x, y, reduction="none").sum(dim=1))
    want = a0 * mult[torch.argmin(torch.stack(losses), dim=0)]
    got = ops.nvfp4_static_mse_sweep(w, a0, g.reshape(1), mult, 256.0)
    n_diff = int((got != want).sum())
    assert n_diff <= 1e-3 * got.numel(), n_diff


# ---- the mirror against the reference's CPU run ----------------------------------------------------------------
def fixture_model(gld, dtype=torch.bfloat16):
    import torch.nn as nn

    class Attn(nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj, self.k_proj = nn.Linear(64, 64, bias=False), nn.Linear(64, 32, bias=False)
            self.v_proj, self.o_proj = nn.Linear(64, 32, bias=False), nn.Linear(64, 48, bias=False)

        def forward(self, x):
            return torch.cat([getattr(self, n)(x) for n in LINEARS], dim=-1)

    m = Attn()
    with torch.no_grad():
        for n in LINEARS:
            getattr(m, n).weight.copy_(torch.from_numpy(gld[f"fos/{n}/w"]))
    return m.to(device="cuda", dtype=dtype)


def test_mirror_quantize_matches_reference_fixture():
    from model_optimizer_b200 import export_hf
    from model_optimizer_b200 import model_quant as mq
    from model_optimizer_b200.config import get_preset

    gld = golden.load("ref_four_over_six")
    model = fixture_model(gld)
    mq.quantize(model, get_preset("NVFP4_FOUR_OVER_SIX_CFG"), None)
    for n in LINEARS:
        wq = getattr(model, n).weight_quantizer
        assert same(wq._amax.cpu().numpy().reshape(-1), gld[f"fos/{n}/amax"]), n
        assert same(wq._global_amax.cpu().numpy(), gld[f"fos/{n}/global_amax"]), n
        t = export_hf.export_linear_tensors(getattr(model, n))
        assert np.array_equal(t["weight"].cpu().numpy(), gld[f"fos/{n}/export/weight"]), n
        assert np.array_equal(t["weight_scale"].view(torch.uint8).cpu().numpy(), gld[f"fos/{n}/export/weight_scale"]), n
        assert same(t["weight_scale_2"].cpu().numpy(), gld[f"fos/{n}/export/weight_scale_2"]), n
    for m in model.modules():
        if hasattr(m, "input_quantizer"):
            m.input_quantizer.disable()
    with torch.no_grad():
        y = model(torch.from_numpy(gld["fos/x"]).cuda().to(torch.bfloat16)).float().cpu().numpy()
    # the fake-quantized weights are bit-equal (above); the bf16 GEMM itself runs on a different device
    assert np.allclose(y, gld["fos/y"], rtol=2e-2, atol=2e-2)


def test_mirror_mse39_matches_reference_fixture():
    import torch.nn as nn

    from model_optimizer_b200 import model_quant as mq
    from model_optimizer_b200.config import get_preset

    gld = golden.load("ref_four_over_six")
    lin = nn.Sequential(nn.Linear(96, 40, bias=False))
    with torch.no_grad():
        lin[0].weight.copy_(torch.from_numpy(gld["mse39/w"]))
    lin = lin.cuda()
    cfg = get_preset("NVFP4_W4A4_WEIGHT_MSE_FP8_SWEEP_CFG")
    cfg["algorithm"] = {"method": "mse"}
    mq.quantize(lin, cfg, None)
    # the fixture's losses were summed in ATen's CPU order and its multipliers built by torch on the CPU; here both
    # are the GPU's: the oracle in the CUDA order with the device's linspace is the bar, and the CPU result agrees
    # wherever the two orders agree
    got = lin[0].weight_quantizer._amax.cpu().numpy().reshape(-1)
    mult = torch.linspace(0.25, 4.0, 39, device="cuda").cpu().numpy()
    want, _, _ = mo.search(gld["mse39/w"], gld["mse39/amax0"], gld["mse39/global_amax"], mult, 448.0, "cuda")
    assert same(got, want)
    assert np.mean(bits(got) == bits(gld["mse39/amax"])) >= 0.99


def test_fp8_scale_sweep_ignores_four_over_six():
    """mse_calibrate(fp8_scale_sweep=True) on a 4/6 quantizer sweeps like any static NVFP4 weight (the reference's
    sweep does not read the normalization); only the later fake quant / export use 256."""
    from model_optimizer_b200 import model_quant as mq
    from model_optimizer_b200.config import get_preset

    gld = golden.load("ref_four_over_six")
    amaxes = []
    for four_over_six in (False, True):
        cfg = get_preset("NVFP4_FOUR_OVER_SIX_CFG")
        cfg["quant_cfg"][1]["cfg"]["block_sizes"]["four_over_six"] = four_over_six
        cfg["algorithm"] = {"method": "mse", "fp8_scale_sweep": True}
        model = fixture_model(gld)
        mq.quantize(model, cfg, None)
        amaxes.append(torch.cat([getattr(model, n).weight_quantizer._amax.reshape(-1) for n in LINEARS]))
    assert torch.equal(amaxes[0], amaxes[1])


# ---- the drop-in against stock mtq.quantize -----------------------------------------------------------------------
def test_dropin_four_over_six():
    from baseline import ref_env

    if not ref_env.available():
        pytest.skip("the reference is not installed (baseline/_ref)")
    mtq = ref_env.activate()
    ref_env.use_prebuilt_extensions()
    from modelopt.torch.export import quant_utils as qu

    from model_optimizer_b200 import backend

    gld = golden.load("ref_four_over_six")
    base = fixture_model(gld)
    x = torch.from_numpy(gld["fos/x"]).cuda().to(torch.bfloat16)
    backend.uninstall()
    stock = mtq.quantize(copy.deepcopy(base), copy.deepcopy(mtq.NVFP4_FOUR_OVER_SIX_CFG), None)
    backend.install()
    backend.stats.clear()
    try:
        mine = mtq.quantize(copy.deepcopy(base), backend.with_b200_backend(mtq.NVFP4_FOUR_OVER_SIX_CFG), None)
        st = dict(backend.stats)
        assert st.get("calib.mse", 0) == len(LINEARS), st
        diff = 0
        for n in LINEARS:
            a, b = getattr(stock, n).weight_quantizer, getattr(mine, n).weight_quantizer
            assert torch.equal(a._global_amax, b._global_amax), n
            diff += int((a._amax != b._amax).sum())
            ta = [qu.get_weight_scaling_factor(getattr(stock, n)), qu.get_weight_scaling_factor_2(getattr(stock, n))]
            tb = [qu.get_weight_scaling_factor(getattr(mine, n)), qu.get_weight_scaling_factor_2(getattr(mine, n))]
            if torch.equal(a._amax, b._amax):
                assert all(torch.equal(p.view(torch.uint8) if p.dtype == torch.float8_e4m3fn else p,
                                       q.view(torch.uint8) if q.dtype == torch.float8_e4m3fn else q)
                           for p, q in zip(ta, tb)), n
        # the stock arm's Triton static kernel rounds a few exact E2M1 ties differently (see above)
        assert diff <= 2, diff
        with torch.no_grad():
            ys, ym = stock(x).float(), mine(x).float()
        assert torch.allclose(ys, ym, rtol=2e-2, atol=2e-2)
    finally:
        backend.uninstall()
