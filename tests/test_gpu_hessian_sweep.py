"""The Hessian-weighted NVFP4 FP8-scale sweep (``b200q_nvfp4_fp8_scale_sweep_hessian``) against its exact CPU oracle
(tools/hessian_sweep_oracle.c) bit for bit, the candidates ``ops`` builds for it, its argument checks, and
``local_hessian_calibrate`` end to end: with the FP8 sweep (the kernel) and without it (the multiplier search under
the Hessian metric, against the reference's CPU run in tests/golden/ref_hessian_sweep.npz)."""

import copy

import numpy as np
import pytest
import torch
from torch import nn
from torch.profiler import ProfilerActivity, profile

import _dispatch_ledger as ledger
from oracle import golden
from oracle import oracle_np as o
from tools import hessian_sweep_oracle as hso

pytestmark = pytest.mark.gpu
TD = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}
ES = {"bf16": 2, "f16": 2, "f32": 4}
DTYPES = ("bf16", "f16", "f32")
NEAR_TIE = 2.0 ** -20
SEEN: set = set()                     # canonical names of the library kernels the profiled calls launched
HERE = ledger.HESSIAN_T


@pytest.fixture(scope="module")
def ops():
    from model_optimizer_b200 import ops as _ops

    return _ops


def same(got, want, what):
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    ok = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    if not ok.all():
        i = int(np.flatnonzero(~ok)[0])
        raise AssertionError(f"{what}: {int((~ok).sum())}/{ok.size} differ, first block {i}: {got.flat[i]!r} vs "
                             f"{want.flat[i]!r}")


def place(a, d, residue=0):
    """``a`` as a contiguous CUDA tensor of dtype ``d`` with ``data_ptr() % 32 == residue``."""
    a = np.ascontiguousarray(a, dtype=np.float32)
    buf = torch.zeros(a.size + 64 // ES[d], dtype=TD[d], device="cuda")
    off = ((residue - buf.data_ptr()) % 32) // ES[d]
    t = buf[off: off + a.size].view(a.shape)
    t.copy_(torch.from_numpy(a).to(TD[d]))
    assert t.data_ptr() % 32 == residue
    return t


def weights(shape, d, seed, scale=0.05):
    """Gaussian with heavy-tailed outliers; in 16-element blocks: all zeros, -0.0, exact E2M1 ties at the
    power-of-two candidate scales of a unit global amax (which one element pins), and zeros of both signs mixed in."""
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(shape) * scale * (1 + 20 * (rng.random(shape) < 1e-2))).astype(np.float32)
    x = np.clip(x, -0.99, 0.99)
    flat = x.reshape(-1)
    flat[0] = 1.0
    nb = flat.size // 16
    ties = np.array([0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, 0.5] * 2, np.float32)
    ties[1::2] *= -1
    mixed = rng.standard_normal(16).astype(np.float32) * np.float32(scale)
    mixed[::3] = -0.0
    mixed[1::5] = 0.0
    special = [np.zeros(16, np.float32), np.full(16, -0.0, np.float32), ties * np.float32(0.125),
               ties * np.float32(0.0625), ties * np.float32(0.03125), mixed]
    if nb > 1:
        pick = rng.choice(np.arange(1, nb), size=min(nb - 1, max(len(special), nb // 16)), replace=False)
        for i, b in enumerate(pick):
            flat[b * 16:(b + 1) * 16] = special[i % len(special)]
    return o.round_to(x, d)


def hessians(n_cin, seed):
    """Per cin block: a positive semi-definite X^T X / n of its own scale, every seventh block from the fourth on
    all zero, every seventh from the sixth on indefinite (random symmetric)."""
    rng = np.random.default_rng(seed)
    h = np.empty((n_cin, 16, 16), np.float32)
    for j in range(n_cin):
        if j % 7 == 3:
            h[j] = 0
        elif j % 7 == 5:
            a = rng.standard_normal((16, 16))
            h[j] = (a + a.T) / 2
        else:
            a = rng.standard_normal((16, 24)) * (1 + 3 * rng.random(16))[:, None] * 10.0 ** rng.uniform(-1, 1)
            h[j] = a @ a.T / 24
    return h


def candidates(ops, spec):
    """The candidate tensor ``ops.nvfp4_fp8_scale_sweep`` sweeps for ``candidates=spec``."""
    if spec == "device":
        return ops.fp8_scale_candidates("cuda")
    if spec == "ieee":
        return ops.fp8_scale_candidates("cpu").cuda()
    return spec


def oracle(ops, w, h, g, spec):
    scales, amaxes = ops.hessian_sweep_candidates(torch.tensor([g], device="cuda"), candidates(ops, spec))
    return hso.hessian_sweep(w.reshape(w.shape[0], -1), h, scales.cpu().numpy(), amaxes.cpu().numpy())


def kernel(ops, w, d, h, spec="device", residue=0, g=None):
    g = np.float32(np.abs(w[np.isfinite(w)]).max(initial=0)) if g is None else np.float32(g)
    got = ops.nvfp4_fp8_scale_sweep(place(w, d, residue), torch.tensor([g], device="cuda"), candidates=spec,
                                    hessian=torch.from_numpy(h).cuda())
    return got.cpu().numpy(), g


def profiled(fn, tries=4):
    """``fn()`` under the CUDA profiler, repeated while a session delivers no kernel record (it now and then
    does not); the library kernels seen go to SEEN."""
    for _ in range(tries):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = fn()
            torch.cuda.synchronize()
        names = {ledger.canonical(e.name) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA}
        names = {n for n in names if n.startswith("b200q::")}
        SEEN.update(names)
        if any(n.startswith("b200q::fp8_sweep_hessian_kernel") for n in names):
            break
    return res


# ---- the kernel against the oracle ---------------------------------------------------------------------------------
@pytest.mark.parametrize("d", DTYPES)
def test_kernel_vs_oracle_shapes(ops, d):
    """cout on and around the 256-row CTA tile times n_cin from one block to a 14336-wide row, 32-byte aligned
    (and 16-byte aligned for the tile-boundary shapes), with zero and indefinite Hessian blocks among them."""
    for cout in (1, 255, 256, 257, 1000):
        for n_cin in (1, 3, 32, 896):
            if n_cin == 896 and cout in (255, 256, 1000):
                continue                                   # the row tail and the wide row: 1 and 257 cover both
            w = weights((cout, n_cin * 16), d, cout * 1000 + n_cin)
            h = hessians(n_cin, n_cin)
            residues = (0, 16) if cout in (255, 257) and n_cin in (3, 32) else (0,)
            for r in residues:
                got, g = (profiled(lambda: kernel(ops, w, d, h, residue=r)) if cout == 257 and n_cin == 3
                          else kernel(ops, w, d, h, residue=r))
                same(got, oracle(ops, w, h, g, "device"), f"{d} cout={cout} n_cin={n_cin} x%32={r}")


@pytest.mark.parametrize("shape", [(4096, 4096), (14336, 4096), (4096, 14336)])
def test_kernel_vs_oracle_llm_weights(ops, shape):
    """bf16 Llama-3-8B weight shapes; the oracle checks the first and last 64 rows and 64 rows between (every cin
    block of each)."""
    cout, cin = shape
    w = weights(shape, "bf16", cout + cin)
    h = hessians(cin // 16, cin)
    got, g = kernel(ops, w, "bf16", h)
    rng = np.random.default_rng(0)
    rows = np.unique(np.concatenate([np.arange(64), np.arange(cout - 64, cout), rng.choice(cout, 64, replace=False)]))
    want = oracle(ops, w[rows], h, g, "device")
    same(got.reshape(cout, -1)[rows].reshape(-1), want, f"bf16 {shape}")


@pytest.mark.parametrize("d", DTYPES)
def test_kernel_candidate_sets(ops, d):
    """``"device"``, ``"ieee"``, one candidate and the 128-candidate maximum (duplicated scales included: the first
    wins), at 32- and 16-byte placement."""
    rng = np.random.default_rng(5)
    w = weights((300, 48), d, 7)
    h = hessians(3, 3)
    many = torch.from_numpy(np.sort(rng.uniform(0.01, 1.0, 128)).astype(np.float32)).cuda()
    many[40:44] = many[40]                                     # equal candidates: equal losses
    for spec in ("device", "ieee", torch.tensor([0.7], device="cuda"), many):
        for r in (0, 16):
            got, g = kernel(ops, w, d, h, spec, r)
            same(got, oracle(ops, w, h, g, spec), f"{d} candidates {spec if isinstance(spec, str) else spec.numel()}")


@pytest.mark.parametrize("d", DTYPES)
def test_kernel_special_values(ops, d):
    """Every candidate scale 0 (global amax < 6 * 2^-24, so s = 1); NaN and inf weights; NaN and inf in the
    Hessian; and for fp32, weights near 1e-12 and 1e30, whose scales leave the reciprocal window (the __fdiv_rn
    path) and whose losses overflow to inf."""
    h = hessians(3, 11)
    tiny = (weights((64, 48), d, 1) * np.float32(2.0 ** -22)).astype(np.float32)
    tiny = o.round_to(np.clip(tiny, -5 * 2.0 ** -24, 5 * 2.0 ** -24), d)
    g = np.float32(np.abs(tiny).max())
    assert 0 < g < 6 * 2.0 ** -24
    scales, _ = ops.hessian_sweep_candidates(torch.tensor([g], device="cuda"), ops.fp8_scale_candidates("cuda"))
    assert torch.all(scales == 0)
    got, g = kernel(ops, tiny, d, h)
    same(got, oracle(ops, tiny, h, g, "device"), f"{d} all scales 0")
    zero = np.zeros((8, 48), np.float32)                       # g = 0: every candidate amax and scale 0
    got, g = kernel(ops, zero, d, h)
    same(got, oracle(ops, zero, h, g, "device"), f"{d} zero weight")
    assert np.all(got == 0)
    w = weights((64, 48), d, 2)
    w[3, 5], w[7, 20], w[9, 40], w[11, 0:16] = np.nan, np.inf, -np.inf, np.nan
    got, g = kernel(ops, w, d, h)
    same(got, oracle(ops, w, h, g, "device"), f"{d} NaN / inf weights")
    hb = h.copy()
    hb[1, 2, 3], hb[2, 7, 7] = np.nan, np.inf
    w = weights((64, 48), d, 3)
    got, g = kernel(ops, w, d, hb)
    same(got, oracle(ops, w, hb, g, "device"), f"{d} NaN / inf Hessian")
    if d == "f32":
        for s in (1e-12, 1e30):
            w = (weights((64, 48), d, 4) * np.float32(s)).astype(np.float32)
            got, g = kernel(ops, w, d, h)
            same(got, oracle(ops, w, h, g, "device"), f"f32 weights near {s}")
        _, losses = hso.hessian_sweep(w[:4], h, *[t.cpu().numpy() for t in ops.hessian_sweep_candidates(
            torch.tensor([g], device="cuda"), ops.fp8_scale_candidates("cuda"))], return_losses=True)
        assert np.isinf(losses).any()                          # the 1e30 case reaches inf losses


def test_candidate_construction(ops):
    """The candidates ``ops`` builds equal a torch restatement of nvfp4_fp8_sweep.py:272-275 on the same device:
    ``amax = c * g`` and ``compute_fp4_scales``'s FP8 fake quant (the CUDA extension's ``fake_e4m3fy``: amax <=
    2^-24 -> 1, then ``448.f / amax`` and ``1.f / scale``, which in C++ ATen are ``fill(...).div_(...)``, IEEE
    divisions, not Python's reciprocal-and-multiply), including g = 0."""
    for g in (0.0, 2.0 ** -26, 1e-12, 0.37, 1.0, 3.0e4, 2.5e38):
        for c in (ops.fp8_scale_candidates("cuda"), ops.fp8_scale_candidates("cpu").cuda()):
            gt = torch.tensor(g, dtype=torch.float32, device="cuda")
            amaxes = c.to(torch.float32) * gt
            q_amax = gt * (448.0 / 448.0) / 6.0
            safe = torch.where(q_amax <= 1.0 / (1 << 24), torch.ones_like(q_amax), q_amax)
            scale = torch.full_like(safe, 448.0).div_(safe)
            inv = torch.ones_like(scale).div_(scale)
            want = ((amaxes / 6.0) * scale).to(torch.float8_e4m3fn).to(torch.float32) * inv
            got_s, got_a = ops.hessian_sweep_candidates(gt.reshape(1), c)
            same(got_a.cpu().numpy(), amaxes.cpu().numpy(), f"cand_amaxes g={g}")
            same(got_s.cpu().numpy(), want.cpu().numpy(), f"cand_scales g={g}")


def test_argument_checks(ops):
    w = weights((32, 48), "bf16", 9)
    h = torch.from_numpy(hessians(3, 9)).cuda()
    g = torch.tensor([1.0], device="cuda")
    for cand in (torch.empty(0, device="cuda"), torch.rand(129, device="cuda")):
        with pytest.raises(ops.B200QuantError):
            ops.nvfp4_fp8_scale_sweep(place(w, "bf16"), g, candidates=cand, hessian=h)
    for d in ("bf16", "f32"):                                  # 8-byte but not 16-byte aligned
        with pytest.raises(ops.B200QuantError):
            ops.nvfp4_fp8_scale_sweep(place(w, d, 8), g, hessian=h)
    for bad in (h[:, :, :8], h[0], h.reshape(3, 16, 16, 1)):
        with pytest.raises(ops.B200QuantError):
            ops.nvfp4_fp8_scale_sweep(place(w, "bf16"), g, hessian=bad)
    with pytest.raises(ops.B200QuantError):                    # 96 blocks over 5 cin blocks
        ops.nvfp4_fp8_scale_sweep(place(w, "bf16"), g, hessian=torch.zeros(5, 16, 16, device="cuda"))


# ---- local_hessian_calibrate ------------------------------------------------------------------------------------------
class _Net(nn.Module):
    """The config-1 MLP (64 -> 128 -> 32, seed 1) and a linear the forward never reaches."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(1)
        self.mlp = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 32))
        self.unused = nn.Linear(64, 32)

    def forward(self, x):
        return self.mlp(x)


def _data(dtype):
    gen = torch.Generator().manual_seed(7)
    return [torch.randn(16, 64, generator=gen).to(dtype).cuda() for _ in range(4)]


def test_local_hessian_fp8_sweep_end_to_end(ops):
    """NVFP4_W4A4_WEIGHT_LOCAL_HESSIAN_CFG (debug) on the config-1 MLP in bf16: each stored Hessian is the restated
    accumulation of the linear's inputs bit for bit, each weight amax is the oracle's sweep under that Hessian with
    the ``ops`` candidates bit for bit, and the linear the forward never reaches gets the plain sweep."""
    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_quant import quantize

    model = _Net().cuda().to(torch.bfloat16)
    data = _data(torch.bfloat16)

    def loop(m):
        for x in data:
            m(x)

    cfg = copy.deepcopy(cfgs.NVFP4_W4A4_WEIGHT_LOCAL_HESSIAN_CFG)
    cfg["algorithm"] = dict(cfg["algorithm"], debug=True)
    profiled(lambda: quantize(model, cfg, loop))
    acc = model._local_hessian_accumulators
    lins = [model.mlp[0], model.mlp[2]]
    assert set(acc) == {id(m.weight_quantizer) for m in lins}
    inputs = {id(m): [] for m in lins}
    hooks = [m.register_forward_pre_hook(lambda m, a: inputs[id(m)].append(a[0].detach().clone())) for m in lins]
    for m in lins:
        m.weight_quantizer.disable()
    try:
        with torch.no_grad():
            loop(model)
    finally:
        for hk in hooks:
            hk.remove()
        for m in lins:
            m.weight_quantizer.enable()
    for m in lins:
        cin = m.weight.shape[1]
        hsum = None
        for x in inputs[id(m)]:                                # _LocalHessianAccumulator.accumulate, restated
            xt = x.reshape(-1, cin).float().T.reshape(cin // 16, 16, -1)
            hb = xt @ xt.transpose(-1, -2)
            hsum = hb if hsum is None else hsum + hb
        want_h = hsum / sum(x.numel() // cin for x in inputs[id(m)])
        e = acc[id(m.weight_quantizer)]
        got_h = e[0] / e[1]
        same(got_h.cpu().numpy(), want_h.cpu().numpy(), f"Hessian of {cin}-wide linear")
        q = m.weight_quantizer
        g = float(q._global_amax)
        want = oracle(ops, m.weight.detach().float().cpu().numpy(), got_h.cpu().numpy(), g, "device")
        same(q._amax.float().cpu().numpy().reshape(-1), want, f"amax of {cin}-wide linear")
    q = model.unused.weight_quantizer
    plain = ops.nvfp4_fp8_scale_sweep(model.unused.weight.contiguous(), q._global_amax.reshape(1))
    same(q._amax.float().cpu().numpy().reshape(-1), plain.cpu().numpy(), "unreached linear")


@pytest.fixture(scope="module")
def ref():
    return golden.load("ref_hessian_sweep")


def _fixture_model(ref, key, dtype):
    model = nn.Sequential(nn.Linear(64, 128), nn.ReLU(), nn.Linear(128, 32))
    with torch.no_grad():
        for li in (0, 2):
            model[li].weight.copy_(torch.from_numpy(ref[f"{key}/l{li}/w"]))
            model[li].bias.copy_(torch.from_numpy(ref[f"{key}/l{li}/b"]))
    data = [torch.from_numpy(x).to(dtype).cuda() for x in ref[f"{key}/data"]]
    return model.cuda().to(dtype), (lambda m: [m(x) for x in data])


def _slot_loss64(q, w, amax, hess):
    """Float64 ``sum dw^T H dw`` per amax slot of ``q`` (dw from the quantizer's own fake quant at ``amax``) and the
    bound ``sum |dw_b H_bd dw_d|`` of its fp32 rounding."""
    from model_optimizer_b200.model_calib import _mse_quant_func

    x = w.detach().float()
    dw = (x - _mse_quant_func(x, amax.reshape(q._amax.shape).to(q._amax.dtype), q)).double()
    dw = dw.view(x.shape[0], -1, 16)
    h = hess.double()
    loss = torch.einsum("cnb,nbd,cnd->cn", dw, h, dw)
    bound = torch.einsum("cnb,nbd,cnd->cn", dw.abs(), h.abs(), dw.abs())
    if q._amax.numel() == 1:
        return loss.sum().reshape(1), bound.sum().reshape(1)
    return loss.sum(1), bound.sum(1)


def _agree(q, w, got, want, hess, what):
    """``got`` equals ``want`` except in slots whose two losses are within fp32 summation error; returns their count."""
    off = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    if off.size:
        lg, bg = _slot_loss64(q, w, torch.from_numpy(got).cuda(), hess)
        lw, bw = _slot_loss64(q, w, torch.from_numpy(want).cuda(), hess)
        gap = (lg - lw).abs().cpu().numpy()[off]
        tol = NEAR_TIE * torch.maximum(bg, bw).cpu().numpy()[off]
        assert np.all(gap <= tol), (what, off[gap > tol][:8], got[off][:8], want[off][:8])
    return off.size


@pytest.mark.parametrize("cname", ["INT8_DEFAULT_CFG", "FP8_DEFAULT_CFG"])
@pytest.mark.parametrize("d", ["f32", "bf16"])
def test_multiplier_search_under_hessian_vs_reference(ref, cname, d):
    """``local_hessian`` with ``fp8_scale_sweep=False`` (INT8 per-channel and FP8 per-tensor weights) against the
    reference's CPU run: the search under the reference's own Hessian with its CPU candidate rule equals it except
    at certified near-ties; the end-to-end run moves the amaxes off max calibration, and in fp32 (where the
    candidate rule is the same on both devices) it equals the reference too."""
    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_calib import _hessian_mse_search_weight
    from model_optimizer_b200.model_quant import quantize

    key, dtype = f"mult/{cname}/{d}", TD[d]
    cfg_max = copy.deepcopy(getattr(cfgs, cname))
    cfg_max["algorithm"] = "max"
    model, loop = _fixture_model(ref, key, dtype)
    quantize(model, cfg_max, loop)
    ties = slots = 0
    for li in (0, 2):
        q, w = model[li].weight_quantizer, model[li].weight
        same(q._amax.float().cpu().numpy().reshape(-1), ref[f"{key}/l{li}/amax_max"].reshape(-1), f"{key} l{li} max")
        hess = torch.from_numpy(ref[f"{key}/l{li}/hess"]).cuda()
        _hessian_mse_search_weight(model[li], hess, 0.1, 0.25, 4.0, round_mult=False)
        got = q._amax.float().cpu().numpy().reshape(-1)
        want = ref[f"{key}/l{li}/amax"].reshape(-1)
        ties += _agree(q, w, got, want, hess, f"{key} l{li} search")
        slots += want.size
    assert ties <= max(1, 0.02 * slots), (ties, slots)

    model, loop = _fixture_model(ref, key, dtype)
    cfg = copy.deepcopy(getattr(cfgs, cname))
    cfg["algorithm"] = {"method": "local_hessian", "fp8_scale_sweep": False, "debug": True}
    quantize(model, cfg, loop)
    acc = model._local_hessian_accumulators
    for li in (0, 2):
        q, w = model[li].weight_quantizer, model[li].weight
        got = q._amax.float().cpu().numpy().reshape(-1)
        amax_max = ref[f"{key}/l{li}/amax_max"].reshape(-1)
        assert np.mean(got != amax_max) > 0.5, (key, li)
        if d == "f32":
            e = acc[id(q)]
            _agree(q, w, got, ref[f"{key}/l{li}/amax"].reshape(-1), e[0] / e[1], f"{key} l{li} end to end")


def test_zz_ledger_variants_ran():
    """Every ledger variant this module covers was launched by a profiled call above."""
    if not SEEN:
        pytest.skip("the profiled cases of this module did not run")
    names = [name for _, name in ledger.variants_for(HERE)]
    assert names
    missing = [n for n in names if not any(ledger.variant_regex(n).match(s) for s in SEEN)]
    assert not missing, (missing, sorted(SEEN))
