"""Input rotation on the GPU: b200q_hadamard bit-exact against the numpy oracle (tools/hadamard_oracle.py) over every
block size, dtype, odd row counts, an unaligned view and inf / NaN / zeros; the folded amax; the fused rotated NVFP4
kernel against the composed three-kernel sequence; autograd; the mirror quantizer against the reference's results
(tests/golden/ref_rotate.npz); and, where the reference is installed, stock mtq.quantize against the drop-in."""

import copy

import numpy as np
import pytest
import torch

from oracle import golden
from tools.hadamard_oracle import hadamard as oracle_hadamard

pytestmark = pytest.mark.gpu

DT = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}


def _bits(t):
    return t.detach().float().cpu().numpy().view(np.uint32)


def _check(x, block, d, amax_slot=None):
    from model_optimizer_b200 import ops

    y = ops.hadamard(x, block, amax_slot)
    want = oracle_hadamard(x.float().cpu().numpy(), block, d)
    got = y.float().cpu().numpy()
    same = (got.view(np.uint32) == want.view(np.uint32)) | (np.isnan(got) & np.isnan(want))
    assert same.all(), (block, d, tuple(x.shape), int((~same).sum()))
    return y


@pytest.mark.parametrize("d", list(DT))
@pytest.mark.parametrize("k", range(16))
def test_hadamard_vs_oracle_all_blocks(k, d):
    b = 1 << k
    g = torch.Generator(device="cuda").manual_seed(k)
    for rows, mult in ((1, 1), (3, 2), (5, 1)):
        if b * mult * rows > (1 << 17):
            rows = 1
        x = torch.randn(rows, b * mult, device="cuda", generator=g).to(DT[d])
        _check(x, b, d)


@pytest.mark.parametrize("d", list(DT))
@pytest.mark.parametrize("dim,block", [(1920, 128), (1536, None), (64, 32), (96, None), (4096, 4096), (24, 8)])
def test_hadamard_shapes_and_wrapper(dim, block, d):
    from model_optimizer_b200.nn.functional import normalized_hadamard_transform, rotate_block_size

    g = torch.Generator(device="cuda").manual_seed(dim)
    x = torch.randn(7, dim, device="cuda", generator=g).to(DT[d])
    b = rotate_block_size(dim, block)
    y = normalized_hadamard_transform(x, block_size=block)
    assert np.array_equal(_bits(y), oracle_hadamard(x.float().cpu().numpy(), b, d).view(np.uint32))
    # rotate_fp32 gives the same bits, and so does transforming the fp32 copy and rounding after
    y32 = normalized_hadamard_transform(x, rotate_fp32=True, block_size=block)
    assert torch.equal(y.view(torch.uint8), y32.view(torch.uint8))
    yf = normalized_hadamard_transform(x.float(), block_size=block).to(x.dtype)
    assert torch.equal(y.view(torch.uint8), yf.view(torch.uint8))


@pytest.mark.parametrize("d", list(DT))
@pytest.mark.parametrize("block", [2, 16, 128, 2048])
def test_hadamard_unaligned_view_and_specials(block, d):
    g = torch.Generator(device="cuda").manual_seed(block)
    base = torch.randn(3 * block * 4 + 1, device="cuda", generator=g).to(DT[d])
    x = base[1:].view(3, block * 4)                        # storage offset of one element: not 32-byte aligned
    assert x.data_ptr() % 32 != 0
    _check(x, block, d)
    s = torch.randn(4, block * 2, device="cuda", generator=g).to(DT[d])
    s[0, 0] = float("inf")
    s[1, 1] = float("nan")
    s[2] = 0.0
    s[3, ::2] = -0.0
    _check(s, block, d)
    odd = torch.randn(block if block < 16 else 1, 6 if block < 16 else block, device="cuda", generator=g).to(DT[d])
    if block < 16:                                          # an element count that is not a multiple of 16
        _check(odd[:, :block * (6 // block)].contiguous(), block, d)


@pytest.mark.parametrize("d", list(DT))
@pytest.mark.parametrize("block", [8, 128, 4096, 32768])
def test_folded_amax_equals_collect(block, d):
    from model_optimizer_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(block + 1)
    for special in (None, "nan", "zeros"):
        x = (torch.randn(4, 32768, device="cuda", generator=g) * 3).to(DT[d])
        if special == "nan":
            x[2, 5] = float("nan")
        elif special == "zeros":
            x.zero_()
        slot = torch.zeros(1, dtype=torch.float32, device="cuda")
        slot.fill_(0.25)                                   # a running max from an earlier batch
        y = _check(x, block, d, slot)
        want = torch.full((1,), 0.25, dtype=torch.float32, device="cuda")
        ops.amax_per_tensor_(want, y)
        assert torch.equal(slot.view(torch.int32), want.view(torch.int32)), (block, d, special, slot, want)


@pytest.mark.parametrize("d", list(DT))
@pytest.mark.parametrize("rotate_back", [False, True])
@pytest.mark.parametrize("shape,block", [((64, 256), 256), ((33, 1920), 128), ((8, 1536), 512), ((16, 4096), 4096),
                                         ((4, 32768), 32768), ((16, 64), 4)])
def test_fused_rotated_nvfp4_equals_composed(shape, block, rotate_back, d):
    from model_optimizer_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(shape[1] + block)
    x = torch.randn(*shape, device="cuda", generator=g).to(DT[d])
    x[0, :16] = 0.0
    x[1, 3] = float("inf")
    r = ops.hadamard(x, block)
    amax = torch.zeros(1, dtype=torch.float32, device="cuda")
    ops.amax_per_tensor_(amax, torch.nan_to_num(r, posinf=0.0))
    amax = amax.to(x.dtype)
    want = ops.fake_quant_nvfp4(r, amax)
    if rotate_back:
        want = ops.hadamard(want, block)
    got = ops.fake_quant_nvfp4_rotated(x, block, amax, rotate_back)
    assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
    xu = torch.cat([x.reshape(-1)[:1], x.reshape(-1)])[1:].view(shape)   # unaligned input
    assert torch.equal(ops.fake_quant_nvfp4_rotated(xu, block, amax, rotate_back).view(torch.uint8),
                       want.view(torch.uint8))


@pytest.mark.parametrize("mode", ["rotate", "rotate_back"])
def test_rotate_backward(mode):
    """test_hadamard.py:116-134: the gradient flows through the rotation (and the rotation back)."""
    from model_optimizer_b200.config import QuantizerAttributeConfig
    from model_optimizer_b200.nn.tensor_quantizer import TensorQuantizer

    q = TensorQuantizer(QuantizerAttributeConfig(num_bits=8, axis=None, rotate={"enable": True, "mode": mode})).cuda()
    x = torch.randn(4, 64, device="cuda", requires_grad=True)
    q.amax = torch.tensor(100.0, device="cuda")          # no clipping: the straight-through gradient is 1
    q(x).sum().backward()
    assert x.grad is not None and torch.isfinite(x.grad).all()
    from model_optimizer_b200 import ops

    ones = torch.ones(4, 64, device="cuda")
    want = ops.hadamard(ones, 64)
    if mode == "rotate_back":
        want = ops.hadamard(want, 64)
    assert torch.equal(x.grad, want)
    # rotated NVFP4 with a calibrated amax keeps its graph (the fused kernel is for no-grad forwards)
    nq = TensorQuantizer(QuantizerAttributeConfig(num_bits=(2, 1), rotate={"enable": True, "mode": mode},
                                                  block_sizes={-1: 16, "type": "dynamic", "scale_bits": (4, 3)})).cuda()
    nq.amax = torch.tensor(4.0, device="cuda")
    x.grad = None
    nq(x).sum().backward()
    assert torch.isfinite(x.grad).all()


def test_quantizer_nvfp4_dispatch_matches_composed(monkeypatch):
    """TensorQuantizer.forward takes the fused NVFP4 branch (once per quantized forward, never while calibrating or
    under autograd), and it gives the bits of the transform + plain fake quant."""
    from model_optimizer_b200 import ops
    from model_optimizer_b200.config import QuantizerAttributeConfig
    from model_optimizer_b200.nn.tensor_quantizer import TensorQuantizer

    fused_calls = []
    fused = ops.fake_quant_nvfp4_rotated

    def spy(*args, **kwargs):
        fused_calls.append(args[1:])
        return fused(*args, **kwargs)

    monkeypatch.setattr(ops, "fake_quant_nvfp4_rotated", spy)
    x = torch.randn(32, 1536, device="cuda").to(torch.bfloat16)
    for mode in ("rotate", "rotate_back"):
        fused_calls.clear()
        q = TensorQuantizer(QuantizerAttributeConfig(num_bits=(2, 1), rotate={"enable": True, "mode": mode},
                                                     block_sizes={-1: 16, "type": "dynamic", "scale_bits": (4, 3)}))
        q.enable_calib()
        q.disable_quant()
        with torch.no_grad():
            q(x)
        assert fused_calls == [], "the calibration pass must not take the fused branch"
        q.load_calib_amax()
        q.disable_calib()
        q.enable_quant()
        with torch.no_grad():
            got = q(x)
        assert len(fused_calls) == 1 and fused_calls[0][0] == 512 and fused_calls[0][2] == (mode == "rotate_back")
        xg = x.float().requires_grad_()                    # an autograd graph: the composed path
        q(xg)
        assert len(fused_calls) == 1
        r = ops.hadamard(x, 512)
        slot = torch.zeros(1, dtype=torch.float32, device="cuda")
        ops.amax_per_tensor_(slot, r)
        assert torch.equal(q.amax.float(), slot.reshape(q.amax.shape))
        want = ops.fake_quant_nvfp4(r, q.amax)
        if mode == "rotate_back":
            want = ops.hadamard(want, 512)
        assert torch.equal(got.view(torch.int16), want.view(torch.int16)), mode


# ---- the mirror against the reference's results ---------------------------------------------------------------------
@pytest.fixture(scope="module")
def ref():
    return golden.load("ref_rotate")


def test_mirror_quantizers_match_reference(ref):
    from model_optimizer_b200.config import QuantizerAttributeConfig
    from model_optimizer_b200.nn.tensor_quantizer import TensorQuantizer

    rotations = {"rot": {"enable": True}, "back": {"enable": True, "mode": "rotate_back"},
                 "fp32b32": {"enable": True, "rotate_fp32": True, "block_size": 32}}
    formats = {"int8": {"num_bits": 8, "axis": None}, "fp8": {"num_bits": (4, 3), "axis": None},
               "int8ch": {"num_bits": 8, "axis": 0}}
    for d, dt in DT.items():
        x = torch.from_numpy(ref[f"tq/{d}/x"]).to(device="cuda", dtype=dt)
        for fname, fcfg in formats.items():
            for rname, rot in rotations.items():
                q = TensorQuantizer(QuantizerAttributeConfig(**fcfg, rotate=rot))
                q.disable_quant()
                q.enable_calib()
                with torch.no_grad():
                    q(x)
                q.load_calib_amax()
                q.disable_calib()
                q.enable_quant()
                key = f"tq/{d}/{fname}/{rname}"
                assert np.array_equal(_bits(q.amax), ref[f"{key}/amax"].view(np.uint32)), key
                with torch.no_grad():
                    assert np.array_equal(_bits(q(x)), ref[f"{key}/y"].view(np.uint32)), key
        for rname, rot in rotations.items():
            q = TensorQuantizer(QuantizerAttributeConfig(num_bits=8, rotate=rot, enable=False))
            assert np.array_equal(_bits(q(x)), ref[f"tq/{d}/disabled/{rname}/y"].view(np.uint32)), (d, rname)


def test_mirror_mlp_matches_reference(ref):
    import model_optimizer_b200.config as cfgs
    from model_optimizer_b200.model_quant import quantize
    from tools.gen_rotate_golden import rotated_inputs

    for d in ("f32", "bf16"):
        key = f"mlp/{d}"
        dt = DT[d]
        model = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 32)).to(dt).cuda()
        with torch.no_grad():
            for i in (0, 2):
                model[i].weight.copy_(torch.from_numpy(ref[f"{key}/w{i}"]).to(dt))
                model[i].bias.copy_(torch.from_numpy(ref[f"{key}/b{i}"]).to(dt))
        data = [torch.from_numpy(ref[f"{key}/calib{i}"]).to(device="cuda", dtype=dt) for i in range(4)]
        with torch.no_grad():
            quantize(model, rotated_inputs(cfgs.INT8_DEFAULT_CFG), lambda m: [m(b) for b in data])
            for i in (0, 2):
                assert np.array_equal(_bits(model[i].input_quantizer.amax), ref[f"{key}/in_amax{i}"].view(np.uint32))
                assert np.array_equal(_bits(model[i].weight_quantizer.amax), ref[f"{key}/w_amax{i}"].view(np.uint32))
            # the GEMMs run on different devices (the fixture's on the CPU), so the logits agree to rounding only
            y, want = model(data[0]).float().cpu().numpy(), ref[f"{key}/logits"]
            assert np.linalg.norm(y - want) <= 1e-2 * np.linalg.norm(want), d


# ---- drop-in: stock mtq.quantize (oracle stand-in for fast_hadamard_transform) vs backend.install() ------------------
def _tiny_llama():
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=2, vocab_size=256, max_position_embeddings=128, tie_word_embeddings=False)
    torch.manual_seed(0)
    return LlamaForCausalLM(cfg).to(device="cuda", dtype=torch.bfloat16).eval()


def _forward_loop(model):
    g = torch.Generator().manual_seed(1)
    for _ in range(4):
        model(torch.randint(0, 256, (2, 48), generator=g).cuda())


def _buffers(model):
    out = {}
    for name, m in model.named_modules():
        if type(m).__name__ == "TensorQuantizer":
            t = getattr(m, "_amax", None)
            if isinstance(t, torch.Tensor):
                out[name] = t.detach().clone()
    return out


@pytest.mark.parametrize("case", ["int8_rotate_inputs", "nvfp4_kv_rotate"])
def test_dropin_rotated_configs(case, monkeypatch):
    import sys

    from baseline import ref_env

    if not ref_env.available():
        pytest.skip("the reference is not installed in baseline/_ref; ref_rotate.npz covers the mirror")
    from tools.gen_rotate_golden import rotated_inputs, stand_in_module

    mtq = ref_env.activate()
    ref_env.use_prebuilt_extensions()
    monkeypatch.setitem(sys.modules, "fast_hadamard_transform", stand_in_module())
    from model_optimizer_b200 import backend

    if case == "int8_rotate_inputs":
        cfg, exact = rotated_inputs(mtq.INT8_DEFAULT_CFG), True
    else:
        cfg, exact = copy.deepcopy(mtq.NVFP4_DEFAULT_CFG), False
        cfg["quant_cfg"] = list(cfg["quant_cfg"]) + copy.deepcopy(list(mtq.NVFP4_KV_ROTATE_CFG["quant_cfg"]))
    base = _tiny_llama()
    backend.uninstall()
    stock = mtq.quantize(copy.deepcopy(base), copy.deepcopy(cfg), _forward_loop)
    backend.install()
    backend.stats.clear()
    try:
        mine = mtq.quantize(copy.deepcopy(base), backend.with_b200_backend(cfg), _forward_loop)
        assert backend.stats["fn.normalized_hadamard_transform"] > 0, dict(backend.stats)
        ids = torch.randint(0, 256, (2, 48), generator=torch.Generator().manual_seed(7)).cuda()
        with torch.no_grad():
            y1 = mine(ids).logits
    finally:
        backend.uninstall()
    with torch.no_grad():
        y0 = stock(ids).logits
    a, b = _buffers(stock), _buffers(mine)
    assert a.keys() == b.keys() and len(a) > 0
    bad = [k for k in a if not torch.equal(a[k], b[k])]
    assert not bad, (case, bad[:6])
    if exact:
        assert torch.equal(y0, y1), (case, float((y0.float() - y1.float()).abs().max()))
    else:                                                  # gross divergence only; the parity bar is per quantizer
        rel = float((y0.float() - y1.float()).norm() / y0.float().norm())
        assert rel < 0.3, (case, rel)
    n_rotated = _rotated_quantizer_outputs(stock, mine, backend, exact, case)
    assert n_rotated > 0, case


def _mismatch(ref, got):
    """(elements that differ, all of them within one code step): the bar of tests/test_gpu_modelopt_dropin.py."""
    ref, got = ref.float(), got.float()
    diff = (ref != got) & ~((ref == 0) & (got == 0))
    r, g = ref[diff].abs(), got[diff].abs()
    hi, lo = torch.maximum(r, g), torch.minimum(r, g)
    return int(diff.sum()), bool(((lo == 0) | (hi / lo <= 2.05)).all())


def _rotated_quantizer_outputs(stock, mine, backend, exact, what):
    """Feed every enabled, rotated quantizer of both arms the same fresh tensor and compare the outputs: bit-equal for
    INT8, and for NVFP4 equal up to exact E2M1 / E4M3 rounding ties (every mismatch within one code step, at most 5 % of
    the elements, as the drop-in file holds the reference's Triton kernels).  Returns the number of quantizers checked."""
    mods0, mods1 = dict(stock.named_modules()), dict(mine.named_modules())
    cfg = stock.config
    head_dim = cfg.hidden_size // cfg.num_attention_heads
    g = torch.Generator(device="cuda").manual_seed(3)
    checked = 0
    for name, q0 in mods0.items():
        if type(q0).__name__ != "TensorQuantizer" or not q0.is_enabled or not q0.rotate_is_enabled:
            continue
        parent = mods0[name.rsplit(".", 1)[0]]
        if hasattr(parent, "in_features"):                 # a linear's input quantizer
            x = torch.randn(2, 48, parent.in_features, device="cuda", generator=g)
        else:                                              # a k / v bmm quantizer: [batch, kv heads, tokens, head dim]
            x = torch.randn(2, cfg.num_key_value_heads, 48, head_dim, device="cuda", generator=g)
        x = (x * 0.7).to(torch.bfloat16)
        with torch.no_grad():
            y0 = q0(x)
            backend.install()
            try:
                y1 = mods1[name](x)
            finally:
                backend.uninstall()
        assert y0.shape == y1.shape and y0.dtype == y1.dtype, (what, name)
        n, bounded = _mismatch(y0, y1)
        if exact:
            assert n == 0, (what, name, n)
        else:
            assert bounded and n <= 0.05 * y0.numel(), (what, name, n, y0.numel())
        checked += 1
    return checked
